"""preprocess.fuse_mc_table and fuse_mesh against the rules and the scalar per-cube loop of include/ofdis_b200.h: the
table's edges, diagonals, sizes and orientation and its committed CUDA copy; the restatement across seeds, odd and thin
shapes and planted values; closed, oriented, edge-manifold meshes on random sign fields and fused volumes; a sampled
sphere and torus; the mesh PLY; and the batch command's --mesh refusals (no device needed)."""
import os
import re

import numpy as np
import pytest

from of_dis_b200 import preprocess

f32 = np.float32
NEXT_BELOW_1 = np.nextafter(f32(1), f32(0))
CORNER = [np.array([q & 1, (q >> 1) & 1, q >> 2]) for q in range(8)]
EDGES = [preprocess.fuse_mc_edge(n) for n in range(12)]


def edge_faces(n):
    q, ax = EDGES[n]
    return {(f, (q >> f) & 1) for f in range(3) if f != ax}


def triangles(tab, case):
    return [tuple(int(v) for v in tab[case, 1 + 3 * t:4 + 3 * t]) for t in range(tab[case, 0])]


# ---- the table -------------------------------------------------------------------------------------------------------
def test_the_table_uses_exactly_the_sign_changing_edges():
    tab = preprocess.fuse_mc_table()
    for case in range(256):
        pos = [(case >> q) & 1 for q in range(8)]
        crossing = {n for n, (q, ax) in enumerate(EDGES) if pos[q] != pos[q | (1 << ax)]}
        used = {v for t in triangles(tab, case) for v in t}
        assert used == crossing, case
        assert tab[case, 0] <= 5 and (tab[case, 1 + 3 * tab[case, 0]:] == 255).all(), case
    assert tab[:, 0].sum() == 820


def test_no_diagonal_lies_on_a_cube_face():
    """A side shared by two triangles of a case is a diagonal: its edges share no cube face.  A side used once is a
    segment of the face rule and lies on a face."""
    tab = preprocess.fuse_mc_table()
    for case in range(256):
        uses = {}
        for t in triangles(tab, case):
            for a, b in ((t[0], t[1]), (t[1], t[2]), (t[2], t[0])):
                uses.setdefault(frozenset((a, b)), []).append((a, b))
        for side, dirs in uses.items():
            a, b = sorted(side)
            if len(dirs) == 1:
                assert edge_faces(a) & edge_faces(b), (case, a, b)
            else:
                assert len(dirs) == 2 and dirs[0] == dirs[1][::-1], (case, dirs)
                assert not edge_faces(a) & edge_faces(b), (case, a, b)


def _edge_mid(n):
    q, ax = EDGES[n]
    return (CORNER[q] + CORNER[q | (1 << ax)]) / 2.0


@pytest.mark.parametrize("q", range(8))
def test_single_corner_cases_face_the_corner(q):
    """One T > 0 corner: the triangle's normal points at it; one T <= 0 corner: away from it."""
    tab = preprocess.fuse_mc_table()
    for case, sign in ((1 << q, 1.0), (255 ^ (1 << q), -1.0)):
        tris = triangles(tab, case)
        assert len(tris) == 1
        p = [_edge_mid(n) for n in tris[0]]
        nrm = np.cross(p[1] - p[0], p[2] - p[0])
        assert sign * np.dot(nrm, CORNER[q] - p[0]) > 0, case


def test_the_boundary_on_each_face_depends_only_on_its_signs():
    """The segments a case leaves on a cube face (sides used once) are a function of that face's four signs: two cubes
    sharing a face meet without cracks."""
    tab = preprocess.fuse_mc_table()
    seen = {}
    for case in range(256):
        sides = {}
        for t in triangles(tab, case):
            for a, b in ((t[0], t[1]), (t[1], t[2]), (t[2], t[0])):
                sides[frozenset((a, b))] = sides.get(frozenset((a, b)), 0) + 1
        for f in range(3):
            for s in (0, 1):
                ring = tuple((case >> q) & 1 for q in range(8) if (q >> f) & 1 == s)
                segs = frozenset(k for k, c in sides.items() if c == 1 and all((f, s) in edge_faces(n) for n in k))
                assert seen.setdefault((f, s, ring), segs) == segs, (case, f, s)


def test_the_committed_cuda_table_equals_the_generator():
    src = open(os.path.join(os.path.dirname(__file__), "..", "of_dis_b200", "csrc", "fusion_kernels.cu")).read()
    body = re.search(r"__constant__ unsigned char FUSE_MC\[256\]\[16\] = \{(.*?)\n\};", src, re.S).group(1)
    rows = re.findall(r"\{([^{}]*)\}", body)
    got = np.array([[int(v) for v in r.split(",")] for r in rows], np.int64)
    assert got.shape == (256, 16)
    assert (got == preprocess.fuse_mc_table()).all()


# ---- the scalar per-cube loop written from the header ----------------------------------------------------------------
def loop_mesh(vol, p, min_weight):
    T, W = vol["T"], vol["W"]
    nz, ny, nx = T.shape
    mw = f32(min_weight)

    def good(k, j, i):
        return W[k, j, i] >= mw and abs(T[k, j, i]) < f32(1)

    vid = {}
    for k in range(nz):
        for j in range(ny):
            for i in range(nx):
                for e, (di, dj, dk) in enumerate(((1, 0, 0), (0, 1, 0), (0, 0, 1))):
                    i2, j2, k2 = i + di, j + dj, k + dk
                    if i2 < nx and j2 < ny and k2 < nz and good(k, j, i) and good(k2, j2, i2) and \
                            (T[k, j, i] > 0) != (T[k2, j2, i2] > 0):
                        vid[(i, j, k, e)] = len(vid)
    tab = preprocess.fuse_mc_table()
    faces = []
    for k in range(nz - 1):
        for j in range(ny - 1):
            for i in range(nx - 1):
                corners = [(i + (q & 1), j + ((q >> 1) & 1), k + (q >> 2)) for q in range(8)]
                if not all(good(c[2], c[1], c[0]) for c in corners):
                    continue
                case = sum(int(T[c[2], c[1], c[0]] > 0) << q for q, c in enumerate(corners))
                for t in range(tab[case, 0]):
                    tri = []
                    for s in range(3):
                        n = int(tab[case, 1 + 3 * t + s])
                        e, r = n >> 2, n & 3
                        q = (r & ((1 << e) - 1)) | ((r >> e) << (e + 1))
                        tri.append(vid[corners[q] + (e,)])
                    faces.append(tri)
    return np.array(faces, np.uint32).reshape(-1, 3), len(vid)


def same(a, b):
    return a.shape == b.shape and np.array_equal(np.ascontiguousarray(a).view(np.uint8),
                                                 np.ascontiguousarray(b).view(np.uint8))


def random_volume(seed, shape, color=1, planted=True):
    """T uniform in (-1.2, 1.2) with planted +0, -0, +-1, nextafter(1, 0), NaN; W in {0, 0.5, nextafter(1, 0), 1, 2}
    and NaN (min_weight 1)."""
    rng = np.random.default_rng(seed)
    nz, ny, nx = shape
    p = dict(nx=nx, ny=ny, nz=nz, origin=(-0.3, 0.1, 0.5), voxel=0.05, trunc=0.15, max_weight=8.0, color=color)
    vol = preprocess.fuse_new_volume(p)
    vol["T"][:] = rng.uniform(-1.2, 1.2, shape).astype(f32)
    vol["W"][:] = rng.choice(np.array([1.0, 2.0, 1.0, 3.0], f32), shape)
    if planted:
        for v, share in ((0.0, 0.05), (-0.0, 0.05), (1.0, 0.02), (-1.0, 0.02), (NEXT_BELOW_1, 0.02),
                         (-NEXT_BELOW_1, 0.02), (np.nan, 0.01)):
            vol["T"][rng.random(shape) < share] = f32(v)
        for v, share in ((0.0, 0.02), (0.5, 0.01), (NEXT_BELOW_1, 0.02), (np.nan, 0.01)):
            vol["W"][rng.random(shape) < share] = f32(v)
    if color:
        vol["C"][:] = rng.integers(0, 256, shape + (3,))
    return vol, p


SHAPES = [(1, 1, 1), (2, 2, 2), (1, 5, 7), (6, 1, 5), (4, 7, 1), (2, 9, 3), (9, 11, 13), (7, 5, 33), (3, 3, 300)]


@pytest.mark.parametrize("seed", [0, 1, 2, 3])
@pytest.mark.parametrize("shape", SHAPES)
def test_restatement_equals_the_loop(seed, shape):
    vol, p = random_volume(100 * seed + sum(shape), shape, color=seed % 2, planted=seed != 3)
    pts, faces = preprocess.fuse_mesh(vol, p, 1.0)
    exp, nv = loop_mesh(vol, p, 1.0)
    assert same(pts, preprocess.fuse_extract(vol, p, 1.0)) and len(pts) == nv
    assert same(faces, exp)
    if min(shape) >= 7:
        assert len(faces) > 10


@pytest.mark.parametrize("mw", [1.0, NEXT_BELOW_1, 2.0])
def test_min_weight_edges(mw):
    """W equal to min_weight passes the test and W just below it fails."""
    vol, p = random_volume(7, (8, 9, 10))
    pts, faces = preprocess.fuse_mesh(vol, p, mw)
    exp, nv = loop_mesh(vol, p, mw)
    assert same(faces, exp) and len(pts) == nv


def test_every_ambiguous_face():
    """Each cube of a 2 x 2 x 2 volume: all 256 cases, the 12 ambiguous faces' two settings among them."""
    tab = preprocess.fuse_mc_table()
    p = dict(nx=2, ny=2, nz=2, origin=(0.0, 0.0, 0.0), voxel=1.0, trunc=1.0, max_weight=2.0, color=0)
    for case in range(256):
        vol = preprocess.fuse_new_volume(p)
        vol["W"][:] = 1
        for q in range(8):
            vol["T"][q >> 2, (q >> 1) & 1, q & 1] = f32(0.5) if (case >> q) & 1 else f32(-0.25)
        pts, faces = preprocess.fuse_mesh(vol, p, 1.0)
        assert len(faces) == tab[case, 0] and same(faces, loop_mesh(vol, p, 1.0)[0]), case


# ---- topology --------------------------------------------------------------------------------------------------------
def check_topology(vol, p, min_weight, pts, faces):
    """Each directed edge at most once; an edge inside the union of meshed cubes once in each direction; indices below
    the vertex count.  Returns the number of interior edges."""
    assert (faces < len(pts)).all()
    T, W = vol["T"], vol["W"]
    nz, ny, nx = T.shape
    good = (W >= f32(min_weight)) & (np.abs(T) < 1)
    meshed = np.zeros((nz + 1, ny + 1, nx + 1), bool)  # padded by one cube at the high ends
    if min(nx, ny, nz) >= 2:
        m = np.ones((nz - 1, ny - 1, nx - 1), bool)
        for q in range(8):
            m &= good[q >> 2:nz - 1 + (q >> 2), (q >> 1) & 1:ny - 1 + ((q >> 1) & 1), q & 1:nx - 1 + (q & 1)]
        meshed[:nz - 1, :ny - 1, :nx - 1] = m
    # each vertex's lattice edge in doubled coordinates (x, y, z): odd along its axis
    idx = np.sort(np.concatenate([np.flatnonzero(_cross(good, T, ax)) * 3 + e for e, ax in ((0, 2), (1, 1), (2, 0))]))
    a, e_of = np.divmod(idx, 3)
    assert len(idx) == len(pts)
    d2 = np.stack([2 * (a % nx), 2 * ((a // nx) % ny), 2 * (a // (nx * ny))], 1)
    d2[np.arange(len(a)), e_of] += 1
    directed = {}
    for t in faces:
        for u, v in ((t[0], t[1]), (t[1], t[2]), (t[2], t[0])):
            assert (u, v) not in directed, "a directed edge used twice"
            directed[(int(u), int(v))] = True
    interior = 0
    for (u, v) in directed:
        du, dv = d2[u], d2[v]
        shared = [f for f in range(3) if du[f] == dv[f] and du[f] % 2 == 0]
        if not shared:
            inside = True  # a diagonal inside one cube
        else:
            f = shared[0]
            c = np.minimum(du // 2, dv // 2)
            lo = c.copy()
            lo[f] = du[f] // 2 - 1
            inside = lo[f] >= 0 and meshed[lo[2], lo[1], lo[0]] and meshed[c[2], c[1], c[0]]
        if inside:
            interior += 1
            assert (v, u) in directed, "an interior edge used in one direction only"
    return interior


def _cross(good, T, ax):
    m = np.zeros(T.shape, bool)
    a = [slice(None)] * 3
    b = [slice(None)] * 3
    a[ax], b[ax] = slice(0, -1), slice(1, None)
    m[tuple(a)] = good[tuple(a)] & good[tuple(b)] & ((T[tuple(a)] > 0) != (T[tuple(b)] > 0))
    return m


@pytest.mark.parametrize("seed", range(4))
def test_random_sign_fields_are_closed_and_oriented(seed):
    rng = np.random.default_rng(seed)
    shape = (9 + seed, 11, 8 + 2 * seed)
    vol, p = random_volume(seed, shape, planted=False)
    vol["T"][:] = np.where(rng.random(shape) < 0.5, f32(0.5), f32(-0.5))
    if seed >= 2:
        vol["W"][rng.random(shape) < 0.1] = 0  # holes: the meshed region gets a boundary
    pts, faces = preprocess.fuse_mesh(vol, p, 1.0)
    assert len(faces) > 200
    assert check_topology(vol, p, 1.0, pts, faces) > 100


def test_fused_volumes_are_closed_and_oriented():
    from test_fusion import CAM, params, scene

    p = params(nx=23, ny=19, nz=21, voxel=0.06)
    disp, poses, frames = scene(3, n=4)
    vol = preprocess.fuse_integrate(preprocess.fuse_new_volume(p), p, disp, poses, CAM, frames=frames)
    pts, faces = preprocess.fuse_mesh(vol, p, 1.0)
    assert len(faces) > 100
    check_topology(vol, p, 1.0, pts, faces)


# ---- analytic shapes -------------------------------------------------------------------------------------------------
def sampled(sdf, n=33, h=0.0625, mu=0.2):
    p = dict(nx=n, ny=n, nz=n, origin=(-1.0, -1.0, -1.0), voxel=h, trunc=mu, max_weight=1.0, color=0)
    xa, ya, za = [np.asarray(a, np.float64) for a in preprocess._fuse_axes(p)]
    Z, Y, X = np.meshgrid(za, ya, xa, indexing="ij")
    vol = preprocess.fuse_new_volume(p)
    vol["T"][:] = np.clip(sdf(X, Y, Z) / mu, -1, 1).astype(f32)
    vol["W"][:] = 1
    return vol, p


def euler(pts, faces):
    edges = {frozenset((int(a), int(b))) for t in faces for a, b in ((t[0], t[1]), (t[1], t[2]), (t[2], t[0]))}
    return len(np.unique(faces)) - len(edges) + len(faces)


def face_normals(pts, faces):
    P = np.stack([pts["x"], pts["y"], pts["z"]], 1).astype(np.float64)
    a, b, c = P[faces[:, 0]], P[faces[:, 1]], P[faces[:, 2]]
    return np.cross(b - a, c - a), (a + b + c) / 3


def test_a_sampled_sphere():
    R = 0.7
    vol, p = sampled(lambda X, Y, Z: np.sqrt(X * X + Y * Y + Z * Z) - R)
    pts, faces = preprocess.fuse_mesh(vol, p, 1.0)
    assert euler(pts, faces) == 2
    check_topology(vol, p, 1.0, pts, faces)
    r = np.sqrt(pts["x"].astype(np.float64) ** 2 + pts["y"] ** 2 + pts["z"] ** 2)
    # linear interpolation of the distance along a lattice edge of h = 0.0625: off by at most h^2 / (2 R) ~ 0.003
    assert np.abs(r - R).max() < 0.005
    n, c = face_normals(pts, faces)
    big = np.linalg.norm(n, axis=1) > 1e-9
    assert big.mean() > 0.99 and (np.einsum("ij,ij->i", n[big], c[big]) > 0).all()


def test_a_sampled_torus():
    vol, p = sampled(lambda X, Y, Z: np.sqrt((np.sqrt(X * X + Z * Z) - 0.6) ** 2 + Y * Y) - 0.25)
    pts, faces = preprocess.fuse_mesh(vol, p, 1.0)
    assert euler(pts, faces) == 0 and len(faces) > 1000
    check_topology(vol, p, 1.0, pts, faces)


def test_write_fused_mesh_ply(tmp_path):
    pts = np.zeros(3, preprocess.FUSE_POINT_DTYPE)
    pts["x"], pts["r"] = (1.5, -2.0, 0.25), (7, 9, 11)
    faces = np.array([[0, 1, 2], [2, 1, 0]], np.uint32)
    path = str(tmp_path / "m.ply")
    preprocess.write_fused_mesh_ply(path, pts, faces)
    head, body = open(path, "rb").read().split(b"end_header\n")
    assert b"element vertex 3" in head and b"element face 2\nproperty list uchar uint vertex_indices\n" in head
    assert len(body) == 3 * 27 + 2 * 13
    rec = np.frombuffer(body[:81], [("p", "<f4", (6,)), ("c", "u1", (3,))])
    assert (rec["p"][:, 0] == pts["x"]).all() and (rec["c"][:, 0] == pts["r"]).all()
    frec = np.frombuffer(body[81:], [("n", "u1"), ("v", "<u4", (3,))])
    assert (frec["n"] == 3).all() and (frec["v"] == faces).all()


# ---- batch command: --mesh is refused where it does not apply (no device needed) -------------------------------------
CAMERA = "721.5,707,16,12,0.54,0.25"
SF = ["--scene-flow", "d.txt", "--camera", CAMERA]
GOOD = "0.1,0.3,-2,-1,1,40,20,60"


def _batch(tmp_path, exe, args):
    from test_fusion import _batch as run

    return run(tmp_path, exe, args)


@pytest.mark.parametrize("exe,args", [
    ("run_OF_INT", ["--mesh"] + SF), ("run_OF_INT", ["--odometry", "odo", "--mesh"] + SF),
    ("run_OF_RGB", ["--mesh"]), ("run_DE_INT", ["--odometry", "odo", "--fuse", GOOD, "--mesh"] + SF),
    ("run_OF_INT", ["--warm-start", "--odometry", "odo", "--fuse", GOOD, "--mesh"] + SF),
    ("run_OF_INT", ["--fuse", GOOD, "--mesh"] + SF),
    ("run_OF_INT", ["--odometry", "odo", "--fuse", "0.1,0.3,-2,-1,1,40,20", "--mesh"] + SF),
    ("run_OF_INT", ["--odometry", "odo", "--mesh", "--fuse", "0.1,0.3,-2,-1,1,1024,1024,1025"] + SF)])
def test_batch_command_refuses_mesh(tmp_path, exe, args):
    r = _batch(tmp_path, exe, args)
    assert r.returncode == 2, (args, r.stdout, r.stderr)


def test_batch_command_accepts_mesh(tmp_path):
    r = _batch(tmp_path, "run_OF_RGB", ["--odometry", "odo", "--mesh", "--fuse", GOOD] + SF)
    assert r.returncode == 0, (r.stdout, r.stderr)
    assert not any(p.name.startswith("fused") for p in (tmp_path / "odo").iterdir())
