"""ofdis_fuse_set_volume and ofdis_fuse_mesh: volumes loaded with set_volume come back bit for bit, and their meshes'
points equal ofdis_fuse_extract and preprocess.fuse_mesh bitwise and their faces exactly (host and device memory, gray
and colour, random fields with planted +-0, +-1, nextafter(1, 0), NaN T and W at and below min_weight, 1x1x1, 2x2x2,
thin and odd shapes whose cubes straddle scan blocks, every case of the table); capacities, fixed launch counts,
argument errors that leave the volume and the outputs, a mesh of synth.rigid_stereo_clip, and the batch command's
--mesh."""
import ctypes
import json
import math

import numpy as np
import pytest

from of_dis_b200 import params, preprocess, synth
from test_fusion_gpu import CAM, SMALL, context, pose, same, scene, vparams
from test_fusion_mesh import NEXT_BELOW_1, check_topology, face_normals, random_volume

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def api():
    from of_dis_b200 import api as _api

    _api.lib()
    return _api


@pytest.fixture(scope="module")
def ctx(api):
    prm = params.from_cli_numbers((SMALL % (1, 0)).split(), noc=1, nop=2)
    c = context(api, prm, 45, 61, 2)
    yield c
    c.close()


def load(ctx, vol, p, memkind, api):
    """fuse_begin(p), then vol through fuse_set_volume from host or device memory."""
    import torch

    ctx.fuse_begin(p)
    if memkind == "host":
        ctx.fuse_set_volume(vol["T"], vol["W"], vol["C"])
    else:
        d = [None if a is None else torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in (vol["T"], vol["W"],
                                                                                             vol["C"])]
        torch.cuda.synchronize()
        ctx.fuse_set_volume(*[None if a is None else a.data_ptr() for a in d], memkind=api.MEM_DEVICE)


def mesh(ctx, api, memkind, mw=1.0, pcap=None, fcap=None):
    """ctx.fuse_mesh through host or device memory: (points, faces, n_points, n_faces)."""
    import torch

    if memkind == "host":
        return ctx.fuse_mesh(mw, pt_capacity=pcap, face_capacity=fcap)
    _, _, nv, nf = ctx.fuse_mesh(mw, memkind=api.MEM_DEVICE)
    pcap = nv if pcap is None else pcap
    fcap = nf if fcap is None else fcap
    # one record more than asked for, with a sentinel: the call must stop at the capacity
    dp = torch.full((28 * (pcap + 1),), 0xAB, dtype=torch.uint8, device="cuda")
    df = torch.full((3 * (fcap + 1),), -7, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    _, _, nv2, nf2 = ctx.fuse_mesh(mw, pt_capacity=pcap, face_capacity=fcap, memkind=api.MEM_DEVICE,
                                   pts_out=dp.data_ptr(), faces_out=df.data_ptr())
    assert (nv2, nf2) == (nv, nf)
    hp, hf = dp.cpu().numpy(), df.cpu().numpy()
    assert (hp[28 * min(pcap, nv):] == 0xAB).all() and (hf[3 * min(fcap, nf):] == -7).all(), "wrote past the total"
    pts = hp[:28 * min(pcap, nv)].view(preprocess.FUSE_POINT_DTYPE)
    return pts, hf[:3 * min(fcap, nf)].view(np.uint32).reshape(-1, 3), nv, nf


def check_mesh(ctx, api, vol, p, mem, mw=1.0, what=""):
    ep, ef = preprocess.fuse_mesh(vol, p, mw)
    gp, gf, nv, nf = mesh(ctx, api, mem, mw)
    assert (nv, nf) == (len(ep), len(ef)), what
    same(gp, ep, what + " points")
    same(gf, ef, what + " faces")
    xp, total = ctx.fuse_extract(mw)
    assert total == nv
    same(gp, xp, what + " points against fuse_extract")
    return ep, ef


@pytest.mark.parametrize("mem", ["host", "device"])
def test_set_volume_round_trip(mem, ctx, api):
    import torch

    for color in (0, 1):
        vol, p = random_volume(5 + color, (13, 17, 19), color=color)
        vol["T"][0, 0, :4] = np.array([np.inf, -np.inf, 3e38, 1e-45], np.float32)
        vol["T"].view(np.uint32)[1, 1, :2] = (0x7FC00001, 0xFFC00000)  # NaN payloads travel as they are
        load(ctx, vol, p, mem, api)
        got = ctx.fuse_volume()
        for k in ("T", "W", "C"):
            same(got[k], vol[k], "%s %d" % (k, color))
        if mem == "device":
            d = {k: torch.empty(vol[k].shape, dtype=torch.float32, device="cuda") for k in ("T", "W")}
            ctx.fuse_volume(memkind=api.MEM_DEVICE, T=d["T"].data_ptr(), W=d["W"].data_ptr())
            for k in ("T", "W"):
                same(d[k].cpu().numpy(), vol[k], "device " + k)
        # NULL arrays keep theirs
        W2 = np.full(vol["W"].shape, 2.5, np.float32)
        if mem == "host":
            ctx.fuse_set_volume(W=W2)
        else:
            dw = torch.from_numpy(W2).cuda()
            torch.cuda.synchronize()
            ctx.fuse_set_volume(W=dw.data_ptr(), memkind=api.MEM_DEVICE)
        got = ctx.fuse_volume()
        same(got["T"], vol["T"], "T after W only")
        same(got["W"], W2, "W after W only")
        same(got["C"], vol["C"], "C after W only")


# (nz, ny, nx): 1x1x1, 2x2x2, one thin in each axis, and odd sizes whose cubes straddle scan blocks of 1024 voxels
SHAPES = [(1, 1, 1), (2, 2, 2), (1, 9, 31), (17, 1, 23), (19, 29, 1), (2, 37, 3), (23, 41, 37), (13, 11, 301),
          (9, 170, 7)]


@pytest.mark.parametrize("mem", ["host", "device"])
@pytest.mark.parametrize("color", [0, 1])
def test_mesh_equals_the_restatement(color, mem, ctx, api):
    for s, shape in enumerate(SHAPES):
        vol, p = random_volume(17 * s + color, shape, color=color)
        load(ctx, vol, p, mem, api)
        for mw in (1.0, float(NEXT_BELOW_1), 2.0):
            ep, ef = check_mesh(ctx, api, vol, p, mem, mw, "%s mw %g" % (shape, mw))
            if min(shape) > 2 and mw == 1.0:
                assert len(ef) > 50, shape
    # a fused volume
    h, w, n = 45, 61, 4
    disp, poses, frames = scene(11, n, h, w, 1)
    p = vparams(color=color)
    vol = preprocess.fuse_integrate(preprocess.fuse_new_volume(p), p, disp, poses, CAM, max_depth=2.5,
                                    frames=frames if color else None)
    load(ctx, vol, p, mem, api)
    ep, ef = check_mesh(ctx, api, vol, p, mem, 1.0, "fused")
    assert len(ef) > 500


def test_every_case_and_ambiguous_face(ctx, api):
    """A 2 x 2 x 2 volume through all 256 cases, at T = +-0.5, and again with the planted +0, -0 and nextafter(1, 0)."""
    p = dict(nx=2, ny=2, nz=2, origin=(0.0, 0.0, 0.0), voxel=1.0, trunc=1.0, max_weight=2.0, color=0)
    tab = preprocess.fuse_mc_table()
    for case in range(256):
        for pos, neg in ((0.5, -0.5), (float(NEXT_BELOW_1), 0.0), (1e-30, -0.0)):
            vol = preprocess.fuse_new_volume(p)
            vol["W"][:] = 1
            for q in range(8):
                vol["T"][q >> 2, (q >> 1) & 1, q & 1] = pos if (case >> q) & 1 else neg
            load(ctx, vol, p, "host", api)
            ep, ef = check_mesh(ctx, api, vol, p, "host", 1.0, "case %d" % case)
            assert len(ef) == tab[case, 0]


@pytest.mark.parametrize("mem", ["host", "device"])
def test_capacities(mem, ctx, api):
    vol, p = random_volume(3, (23, 41, 37), color=1)
    load(ctx, vol, p, mem, api)
    ep, ef = preprocess.fuse_mesh(vol, p, 1.0)
    nv, nf = len(ep), len(ef)
    for pcap in (0, 1, nv - 1, nv, None):
        for fcap in (0, 1, nf - 1, None):
            gp, gf, v, f = mesh(ctx, api, mem, 1.0, pcap, fcap)
            assert (v, f) == (nv, nf)
            same(gp, ep[:nv if pcap is None else pcap], "points at %s" % pcap)
            same(gf, ef[:nf if fcap is None else fcap], "faces at %s" % fcap)


def test_launch_counts(api):
    """Six kernels for a tiny and a large volume; the extraction keeps its three."""
    prm = params.from_cli_numbers((SMALL % (1, 0)).split(), noc=1, nop=2)
    c = context(api, prm, 45, 61, 2)
    import torch

    counts = {}
    dp = torch.empty(28 * 5, dtype=torch.uint8, device="cuda")
    df = torch.empty(15, dtype=torch.int32, device="cuda")
    for name, shape in (("tiny", (2, 2, 2)), ("large", (300, 200, 250))):
        vol, p = random_volume(9, shape, color=0, planted=False)
        load(c, vol, p, "host", api)
        before = c.launch_count
        c.fuse_mesh(1.0, pt_capacity=0, face_capacity=0)
        counts[name + " host count"] = c.launch_count - before
        before = c.launch_count
        c.fuse_mesh(1.0, pt_capacity=5, face_capacity=5, memkind=api.MEM_DEVICE, pts_out=dp.data_ptr(),
                    faces_out=df.data_ptr())
        counts[name + " device"] = c.launch_count - before
        before = c.launch_count
        c.fuse_mesh(1.0, pt_capacity=5, face_capacity=5)
        counts[name + " host"] = c.launch_count - before
        before = c.launch_count
        c.fuse_extract(1.0, capacity=5)
        counts[name + " extract"] = c.launch_count - before
    c.close()
    assert counts == {"tiny host count": 6, "tiny device": 6, "tiny host": 6, "tiny extract": 3,
                      "large host count": 6, "large device": 6, "large host": 6, "large extract": 3}, counts


def test_argument_errors_leave_the_volume_and_the_outputs(api):
    prm = params.from_cli_numbers((SMALL % (1, 0)).split(), noc=1, nop=2)
    c = context(api, prm, 45, 61, 2)
    L = api.lib()
    nv, nf = ctypes.c_long(-3), ctypes.c_long(-3)
    pbuf = np.zeros(4, preprocess.FUSE_POINT_DTYPE)
    pbuf.view(np.uint8)[:] = 0x5A
    fbuf = np.full((4, 3), 77, np.uint32)
    T, W = np.zeros((2, 2, 2), np.float32), np.ones((2, 2, 2), np.float32)

    def m(mw=1.0, P=pbuf, pc=4, pn=True, F=fbuf, fc=4, fn=True, mk=0):
        return L.ofdis_fuse_mesh(c._h, mw, api._ptr(P), pc, ctypes.byref(nv) if pn else None, api._ptr(F), fc,
                                 ctypes.byref(nf) if fn else None, mk)

    errs = [m(), L.ofdis_fuse_set_volume(c._h, api._ptr(T), api._ptr(W), None, 0)]  # no live volume
    vol, p = random_volume(4, (9, 11, 13), color=0)
    load(c, vol, p, "host", api)
    errs += [m(pn=False), m(fn=False), m(pc=-1), m(fc=-1), m(P=None), m(F=None), m(mw=float("nan")),
             m(P=2, mk=1), m(F=2, mk=1), m(P=None, pc=0, F=6, mk=1)]
    errs += [L.ofdis_fuse_set_volume(c._h, None, None, api._ptr(np.zeros(3 * 9 * 11 * 13, np.uint8)), 0),
             L.ofdis_fuse_set_volume(c._h, api._ptr(2), None, None, 1),
             L.ofdis_fuse_set_volume(c._h, None, api._ptr(6), None, 1)]
    assert all(e == -1 for e in errs), errs  # OFDIS_ERR_ARG
    assert nv.value == -3 and nf.value == -3
    assert (pbuf.view(np.uint8) == 0x5A).all() and (fbuf == 77).all()
    got = c.fuse_volume()
    for k in ("T", "W"):
        same(got[k], vol[k], "after the errors: " + k)
    assert m(P=None, pc=0, F=None, fc=0) == 0 and nf.value == len(preprocess.fuse_mesh(vol, p, 1.0)[1])
    c.close()


def test_mesh_of_a_synthetic_rig_clip(api):
    """synth.rigid_stereo_clip at KITTI's size, as tests/test_fusion_gpu.py fuses it (operating point 2, lr-check, 8
    frames, 0.1 m voxels): the mesh is closed and oriented inside the meshed cubes, its face normals agree with the
    extraction's vertex normals, and its ground lies at y = 1.65."""
    h, w, n = 375, 1242, 8
    cam = dict(fx=721.5, fy=721.5, cx=609.6, cy=172.9, baseline=0.54, doffs=0.0)
    rels = [pose((0.0, math.radians(0.3 * (k % 3 - 1)), 0.0), (0.02 * (k % 2), 0.0, -0.5)) for k in range(n - 1)]
    clip = synth.rigid_stereo_clip(n - 1, h, w, 1, 2, cam, rels, block={"velocity": (0.0, 0.0, 0.0)})
    prm = params.operating_point(2, w, noc=1, nop=1)
    c = context(api, prm, h, w, 2 * n)
    fwd = np.stack([clip["left"], clip["right"]], 1)
    c.upload_frames_u8(0, 2 * n, np.ascontiguousarray(np.concatenate([fwd, fwd[:, ::-1]])), w, h)
    c.set_swapped_slots(n, 2 * n, 1)
    c.run(2 * n)
    disp = c.disparity_fullres(0, n, n, w, h, lr_check=1, outputs=("disp",))["disp"]
    p = dict(nx=160, ny=55, nz=280, origin=(-8.0, -3.0, 3.0), voxel=0.1, trunc=0.3, max_weight=64.0, color=0)
    c.fuse_begin(p)
    c.fuse_push(disp, clip["abs"], cam, width_org=w, height_org=h)
    pts, faces, nv, nf = c.fuse_mesh(1.0)
    vol = c.fuse_volume()
    c.close()
    ep, ef = preprocess.fuse_mesh(vol, p, 1.0)
    same(pts, ep, "clip points")
    same(faces, ef, "clip faces")
    check_topology(vol, p, 1.0, pts, faces)
    nrm, cen = face_normals(pts, faces)
    L = np.linalg.norm(nrm, axis=1)
    ok = L > 1e-12
    vn = np.stack([pts["nx"], pts["ny"], pts["nz"]], 1).astype(np.float64)
    mean_vn = np.nan_to_num(vn[faces[ok]]).sum(1)
    agree = np.einsum("ij,ij->i", nrm[ok], mean_vn) > 0
    unit = nrm[ok] / L[ok, None]
    ground = unit[:, 1] < -0.9
    figures = dict(faces=int(nf), vertices=int(nv), nondegenerate=int(ok.sum()), agree_share=float(agree.mean()),
                   ground_faces=int(ground.sum()), ground_median=float(np.median(np.abs(cen[ok][ground, 1] - 1.65))))
    print(json.dumps(figures))
    # bounds written before the first run: nine in ten non-degenerate faces point the way of their vertices' mean
    # extraction normal, and the ground's faces lie within one voxel of y = 1.65 (median)
    assert figures["faces"] > 10000 and figures["nondegenerate"] > 0.9 * figures["faces"], figures
    assert figures["agree_share"] >= 0.9, figures
    assert figures["ground_faces"] > 1000 and figures["ground_median"] < p["voxel"], figures


def test_batch_command_mesh(tmp_path):
    """run_OF_INT_batch --fuse --mesh: each fused_<clip>_mesh.ply equals write_fused_mesh_ply of the restatement on the
    written poses, and fused_<clip>.ply has the same bytes as without --mesh."""
    import subprocess

    from of_dis_b200 import build

    bindir = build.build_host()
    h, w, n = 91, 150, 3
    cam = dict(fx=180.0, fy=176.5, cx=w / 2 - 0.25, cy=h / 2 + 0.5, baseline=0.54, doffs=0.25)
    rels = [pose((0.0, 0.01, 0.0), (0.03, 0.0, -0.5)), pose((0.004, -0.006, 0.002), (0.0, 0.01, -0.3)),
            pose((0.0, 0.0, 0.0), (0.05, 0.0, -0.6))]
    clip = synth.rigid_stereo_clip(n, h, w, 1, 31, cam, rels)
    rng = np.random.default_rng(31)
    maps = clip["disp"].copy()
    maps[rng.random(maps.shape) < 0.03] = np.nan
    for k in range(n + 1):
        preprocess.write_pgm(str(tmp_path / ("f%d.pgm" % k)), clip["left"][k])
        preprocess.write_pfm(str(tmp_path / ("d%d.pfm" % k)), -maps[k])
    pairs = [(k, k + 1) for k in range(n)] + [(2, 0)]
    (tmp_path / "list.txt").write_text("".join("f%d.pgm f%d.pgm out%d.flo\n" % (a, b, j)
                                               for j, (a, b) in enumerate(pairs)))
    (tmp_path / "disps.txt").write_text("".join("d%d.pfm d%d.pfm\n" % ab for ab in pairs))
    camarg = ",".join(repr(float(cam[k])) for k in preprocess.STEREO_CAMERA_FIELDS)
    spec = "0.25,0.75,-6,-3,2,48,20,80"
    out = {}
    for name, extra in (("plain", []), ("mesh", ["--mesh"])):
        (tmp_path / name).mkdir()
        r = subprocess.run([str(bindir) + "/run_OF_INT_batch", "list.txt", "--batch", "2", "--scene-flow", "disps.txt",
                            "--camera", camarg, "--odometry", name, "--fuse", spec] + extra, capture_output=True,
                           text=True, cwd=str(tmp_path))
        assert r.returncode == 0, r.stderr
        out[name] = r.stdout
    p = dict(nx=48, ny=20, nz=80, origin=(-6.0, -3.0, 2.0), voxel=0.25, trunc=0.75, max_weight=64.0, color=1)
    lines = [ln.split() for ln in out["mesh"].splitlines() if ln.startswith("MESH")]
    assert not any(ln.startswith("MESH") for ln in out["plain"].splitlines())
    assert not (tmp_path / "plain" / "fused_0000_mesh.ply").exists()
    for c, frames in ((0, [0, 1, 2, 3]), (1, [2, 0])):
        fused = "fused_%04d.ply" % c
        assert (tmp_path / "mesh" / fused).read_bytes() == (tmp_path / "plain" / fused).read_bytes(), c
        poses = preprocess.read_kitti_poses(str(tmp_path / "mesh" / ("poses_%04d.txt" % c)))
        d = np.stack([-preprocess.read_pfm(str(tmp_path / ("d%d.pfm" % k)))[..., 0] for k in frames])
        vol = preprocess.fuse_integrate(preprocess.fuse_new_volume(p), p, d, poses, cam, max_depth=np.inf,
                                        frames=clip["left"][frames])
        pts, faces = preprocess.fuse_mesh(vol, p, 1.0)
        assert len(faces) > 100
        exp = tmp_path / ("exp%d.ply" % c)
        preprocess.write_fused_mesh_ply(str(exp), pts, faces)
        assert (tmp_path / "mesh" / ("fused_%04d_mesh.ply" % c)).read_bytes() == exp.read_bytes(), c
        assert lines[c] == ["MESH", "clip", str(c), "vertices", str(len(pts)), "faces", str(len(faces))], lines
