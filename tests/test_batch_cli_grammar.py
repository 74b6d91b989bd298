"""The batch command's grammar (run_*_batch of of_dis_b200/host/run_dense.cpp) on CPU: every refusal that comes
before any device work, with its exit code, its whole stderr line and the files it leaves behind; the flag
combinations accepted on an empty list with the exact bytes of every file they write; the usage text."""
import os
import subprocess

import numpy as np
import pytest

from of_dis_b200 import build
from of_dis_b200 import preprocess as pp

FLOW = ["run_OF_INT", "run_OF_RGB"]
STEREO = ["run_DE_INT", "run_DE_RGB"]
ALL = FLOW + STEREO

PAIR = "(binary PGM/PPM or 8-bit PNG of equal size)"
WARM = "error: --warm-start runs one pair per launch; it takes no %s"
CAM = "1,1,0,0,0.5,0"
FUSE = "0.1,0.3,0,0,0,4,4,4"
GM = ["--global-motion", "affine", "gm.txt"]
SF = ["--scene-flow", "empty.txt"]
ODO = SF + ["--camera", CAM, "--odometry", "."]
TRACKS_HDR = b"# clip frame id x y\n"
DESC_HDR = b"# clip id start mean_x mean_y sd_x sd_y length d0 .. d425\n"
FISHER_HDR = b"# clip n_desc n_0 .. n_4 fv0 .. fv%d\n" % (2 * 2 * 213 - 1)  # K 2, every block at half its width

USAGE = (
    "usage: %s listfile [--batch N | --warm-start] [--bidirectional] [--gt gtlist] [--kitti]\n"
    "       [--color [--color-max M]] [--interpolate T]\n"
    "       [--tracks PATH [--descriptors PATH] [--fisher CODEBOOK PATH]]\n"
    "       [--lr-check] [--speckle N R] [--fill] [--camera fx,fy,cx,cy,baseline,doffs]\n"
    "       [--global-motion similarity|affine|homography PATH [--stabilize RADIUS CROP DIR]]\n"
    "       [--scene-flow DISPLIST [--gt-scene-flow GTLIST]]\n"
    "       [--odometry DIR [--gt-poses LIST] [--fuse voxel,trunc,x0,y0,z0,nx,ny,nz [--mesh]]]\n"
    "       [oppoint | 20 parameters (README.md:66-88)]\n"
    "  --warm-start: latency mode for video, one pair per launch; a pair whose image1 is the previous pair's\n"
    "  image2 starts from that pair's flow (the reference's init flow); a clip then runs serially\n"
    "  --bidirectional: also the backward flow (stereo: the right view's disparity) of every pair, written to\n"
    "  <stem>_bw<ext>, and the forward-backward consistency mask to <stem>_occ.pgm (0 consistent,\n"
    "  255 inconsistent, 128 leaves the frame); not with --warm-start\n"
    "  --gt gtlist: ground-truth files (.flo / .pfm, or KITTI's 16-bit PNG), one per pair in list order; prints\n"
    "  EVAL lines (end-point error, shares above 1, 3, 5 px, KITTI outliers; with --bidirectional also per\n"
    "  consistency class)\n"
    "  --kitti: write every flow (and _bw) output as KITTI's 16-bit PNG (flow RGB16, stereo gray16 disparity),\n"
    "  whatever its extension\n"
    "  --color: also write <stem>_color.png (and <stem>_bw_color.png), the 8-bit RGB color coding of every\n"
    "  output (flow: Middlebury's color wheel, stereo: KITTI's disparity colors), colored on the device\n"
    "  --color-max M: color every pair with the scale M (a positive finite number) instead of its own maximum\n"
    "  --interpolate T: also write <stem>_interp.png, the frame at time T (0 < T < 1) between image1 and image2,\n"
    "  synthesised on the device from the forward and backward flows; not with --warm-start\n"
    "  --tracks PATH: dense point trajectories through every clip of the list, written to PATH as lines\n"
    "  `clip frame id x y`; not with --warm-start\n"
    "  --descriptors PATH: flow only, with --tracks; the trajectory descriptors (shape, HOG, HOF, MBH) of every\n"
    "  15-frame segment of the tracks, camera-compensated with the --global-motion models when given, written to\n"
    "  PATH as lines `clip id start mean_x mean_y sd_x sd_y length` and 426 floats; frames of at least 32 x 32;\n"
    "  not with --warm-start\n"
    "  --fisher CODEBOOK PATH: flow only, with --tracks; one Fisher vector per clip of the descriptors above,\n"
    "  encoded on the device with the codebook file CODEBOOK (python -m of_dis_b200.fisher_fit), written to\n"
    "  PATH as lines `clip n_desc n_0 .. n_4` and the vector; not with --warm-start\n"
    "  --lr-check, --speckle N R, --fill, --camera ...: stereo only; also write <stem>_filtered<ext>, the\n"
    "  disparity without the pixels that fail the left-right check and the speckles of at most N pixels (R px),\n"
    "  holes filled with the background disparity, and with --camera <stem>_depth.pfm and <stem>.ply;\n"
    "  not with --warm-start\n"
    "  --global-motion MODEL PATH: flow only; the camera motion of every pair, one line per pair in PATH, and\n"
    "  <stem>_residual<ext>, <stem>_moving.pgm and <stem>_registered.png; not with --warm-start\n"
    "  --stabilize RADIUS CROP DIR: flow only, with --global-motion; every clip stabilised along its smoothed\n"
    "  camera path (RADIUS 1..64 frames each side, CROP 0 <= CROP < 0.5 cut from each side), written to\n"
    "  DIR/stab_<clip>_<frame>.png, the corrections to DIR/stab.txt; not with --warm-start\n"
    "  --scene-flow DISPLIST (flow binaries): the disparities of image1 and image2 of every pair (PFM or KITTI\n"
    "  PNG) give <stem>_disp1.pfm (<stem>_disp1<ext> with --kitti), and with --camera <stem>_sceneflow.pfm;\n"
    "  --gt-scene-flow GTLIST: disp0, disp1 and flow ground truth per pair, SFEVAL lines; not with --warm-start\n"
    "  --odometry DIR (flow binaries, with --scene-flow and --camera): the rig's ego-motion of every pair to\n"
    "  DIR/odometry.txt, each clip's KITTI poses to DIR/poses_<clip>.txt, <stem>_objects.pgm and\n"
    "  <stem>_objmotion.pfm; --gt-poses LIST: one KITTI poses file per clip, ODOEVAL lines; not with --warm-start\n"
    "  --fuse voxel,trunc,x0,y0,z0,nx,ny,nz (flow binaries, with --odometry): every clip's disparities fused\n"
    "  into a TSDF volume of nx x ny x nz voxels from (x0, y0, z0), its surface points to DIR/fused_<clip>.ply;\n"
    "  not with --warm-start\n"
    "  --mesh (with --fuse): also the volume's triangle mesh to DIR/fused_<clip>_mesh.ply\n")


@pytest.fixture(scope="module")
def bindir():
    return build.build_host()


def _codebook(blocks=None):
    rng = np.random.default_rng(0)
    blocks = blocks or [(o, di, di // 2) for o, di in pp.fisher_blocks(pp.TRAJ_DEFAULTS)]
    cb = {"K": 2, "desc_dim": pp.traj_dim(pp.TRAJ_DEFAULTS), "blocks": blocks}
    for k in pp.FISHER_PARTS:
        cb[k] = []
    for _, di, d in blocks:
        w = np.full(2, 0.5)
        cb["mean"].append(rng.normal(0, 0.5, di).astype(np.float32))
        cb["proj"].append(rng.normal(0, 0.1, (d, di)).astype(np.float32))
        cb["mu"].append(rng.normal(0, 1.0, (2, d)).astype(np.float32))
        cb["isig"].append(np.ones((2, d), np.float32))
        cb["c"].append(np.log(w).astype(np.float32))
        cb["w"].append(w.astype(np.float32))
    return cb


def _pgm(path, w, h):
    with open(path, "wb") as f:
        f.write(b"P5\n%d %d\n255\n" % (w, h) + bytes(w * h))


def _pfm(path, w, h):
    with open(path, "wb") as f:
        f.write(b"Pf\n%d %d\n-1.000000\n" % (w, h) + np.full(w * h, -1.0, "<f4").tobytes())


@pytest.fixture
def work(tmp_path):
    """The inputs every case may name, relative to the working directory; returns it and the names it holds."""
    (tmp_path / "list.txt").write_text("")
    (tmp_path / "empty.txt").write_text("")
    (tmp_path / "one.txt").write_text("x\n")
    (tmp_path / "out").mkdir()
    pp.write_fisher_codebook(str(tmp_path / "cb.fv"), _codebook())
    pp.write_fisher_codebook(str(tmp_path / "blocks.fv"), _codebook(blocks=[(0, 30, 15), (30, 396, 8)]))
    (tmp_path / "magic.fv").write_bytes(b"OFDISFV0" + (tmp_path / "cb.fv").read_bytes()[8:])
    _pgm(tmp_path / "a16.pgm", 16, 16)
    _pgm(tmp_path / "b16.pgm", 16, 16)
    _pgm(tmp_path / "a40.pgm", 40, 40)
    _pgm(tmp_path / "b40.pgm", 40, 40)
    _pfm(tmp_path / "d40.pfm", 40, 40)
    _pfm(tmp_path / "d16.pfm", 16, 16)
    (tmp_path / "disp16.txt").write_text("d16.pfm d16.pfm\n")
    (tmp_path / "small.txt").write_text("a16.pgm b16.pgm o.flo\n")
    (tmp_path / "pair40.txt").write_text("a40.pgm b40.pgm o.flo\n")
    (tmp_path / "gone.txt").write_text("nope1.pgm nope2.pgm o.flo\n")
    (tmp_path / "gt_gone.txt").write_text("g.flo\n")
    (tmp_path / "disp40.txt").write_text("d40.pfm d40.pfm\n")
    (tmp_path / "disp40_gone.txt").write_text("d40.pfm gone.pfm\n")
    (tmp_path / "poses.txt").write_text("p0.txt\n")
    (tmp_path / "p0.txt").write_text("1 0 0 0 0 1 0 0 0 0 1 0\n")
    (tmp_path / "poses_gone.txt").write_text("gone_poses.txt\n")
    return tmp_path, {q.name: q.read_bytes() if q.is_file() else None for q in tmp_path.iterdir()}


def _run(bindir, exe, args, cwd):
    return subprocess.run([os.path.join(bindir, exe + "_batch")] + args, capture_output=True, text=True, cwd=str(cwd))


def _written(cwd, inputs):
    """Every file a run added, by path relative to cwd, with its bytes; inputs must keep theirs."""
    out = {}
    for root, _, files in os.walk(cwd):
        for name in files:
            rel = os.path.relpath(os.path.join(root, name), cwd)
            data = open(os.path.join(root, name), "rb").read()
            if rel in inputs:
                assert inputs[rel] == data, rel
            else:
                out[rel] = data
    return out


# (binaries, arguments after the list file, exit code, stderr line, files left behind)
REFUSED = [
    # an argument-taking flag without its arguments, or given twice
    (ALL, ["--color", "--color-max"], 2, "error: --color-max takes one positive number", {}),
    (ALL, ["--color-max", "1", "--color-max", "2"], 2, "error: --color-max takes one positive number", {}),
    (ALL, ["--interpolate"], 2, "error: --interpolate takes one time between 0 and 1", {}),
    (ALL, ["--tracks", "t.txt", "--tracks", "u.txt"], 2, "error: --tracks takes one output path", {}),
    (FLOW, ["--tracks", "t.txt", "--descriptors"], 2, "error: --descriptors takes one output path", {}),
    (FLOW, ["--tracks", "t.txt", "--fisher", "cb.fv"], 2, "error: --fisher takes a codebook file and an output path",
     {}),
    (STEREO, ["--speckle", "5"], 2, "error: --speckle takes a size N and a difference R", {}),
    (STEREO, ["--camera"], 2, "error: --camera takes fx,fy,cx,cy,baseline,doffs", {}),
    (FLOW, ["--global-motion", "affine"], 2,
     "error: --global-motion takes a model (similarity, affine or homography) and an output path", {}),
    (FLOW, GM + ["--stabilize", "4", "0.1"], 2, "error: --stabilize takes a radius, a crop and an output directory",
     {}),
    (FLOW, ["--scene-flow"], 2, "error: --scene-flow takes one disparity list file", {}),
    (FLOW, SF + ["--gt-scene-flow"], 2, "error: --gt-scene-flow takes one ground-truth list file", {}),
    (FLOW, SF + ["--camera", CAM, "--odometry"], 2, "error: --odometry takes one output directory", {}),
    (FLOW, ODO + ["--fuse"], 2, "error: --fuse takes voxel,trunc,x0,y0,z0,nx,ny,nz", {}),
    (FLOW, ODO + ["--gt-poses"], 2, "error: --gt-poses takes one list of KITTI poses files", {}),
    (ALL, ["--gt", "empty.txt", "--gt", "empty.txt"], 2, "error: --gt takes one ground-truth list file", {}),
    # --warm-start
    (ALL, ["--warm-start", "--batch", "4"], 2, WARM % "--batch", {}),
    (ALL, ["--warm-start", "--bidirectional"], 2, WARM % "--bidirectional", {}),
    (ALL, ["--warm-start", "--interpolate", "0.5"], 2, WARM % "--interpolate", {}),
    (ALL, ["--warm-start", "--tracks", "t.txt"], 2, WARM % "--tracks", {}),
    (FLOW, ["--warm-start"] + SF, 2, WARM % "--scene-flow", {}),
    (FLOW, ["--warm-start", "--odometry", "."], 2, WARM % "--odometry", {}),
    (FLOW, ["--warm-start", "--fuse", FUSE], 2, WARM % "--fuse", {}),
    (STEREO, ["--warm-start", "--fill"], 2, WARM % "--lr-check, --speckle, --fill or --camera", {}),
    (FLOW, ["--warm-start"] + GM, 2, WARM % "--global-motion", {}),
    (FLOW, ["--warm-start", "--descriptors", "d.txt"], 2, WARM % "--descriptors", {}),
    (FLOW, ["--warm-start", "--fisher", "cb.fv", "f.txt"], 2, WARM % "--fisher", {}),
    (FLOW, ["--warm-start", "--stabilize", "4", "0.1", "out"], 2, WARM % "--stabilize", {}),
    # the flags of one kind of binary
    (STEREO, SF, 2, "error: --scene-flow joins flows with disparities; the stereo binaries take no --scene-flow", {}),
    (STEREO, ["--odometry", "."], 2,
     "error: --odometry fits the rig's motion from flows; the stereo binaries take no --odometry", {}),
    (STEREO, ["--fuse", FUSE], 2,
     "error: --fuse places disparities with the poses of --odometry; the stereo binaries take no --fuse", {}),
    (FLOW, ["--lr-check"], 2, "error: --lr-check, --speckle, --fill and --camera filter stereo disparities; the flow "
     "binaries take none of them", {}),
    (FLOW, ["--camera", CAM], 2, "error: --lr-check, --speckle, --fill and --camera filter stereo disparities; the "
     "flow binaries take none of them", {}),
    (STEREO, GM, 2, "error: --global-motion fits the camera motion of flows; the stereo binaries take no "
     "--global-motion", {}),
    (STEREO, ["--tracks", "t.txt", "--descriptors", "d.txt"], 2,
     "error: --descriptors describes the tracks of flows; the stereo binaries take no --descriptors", {}),
    (STEREO, ["--tracks", "t.txt", "--fisher", "cb.fv", "f.txt"], 2,
     "error: --fisher encodes the descriptors of flows; the stereo binaries take no --fisher", {}),
    (STEREO, ["--stabilize", "4", "0.1", "out"], 2,
     "error: --stabilize smooths the camera motion of flows; the stereo binaries take no --stabilize", {}),
    # a flag that needs another
    (FLOW, ["--gt-scene-flow", "empty.txt"], 2,
     "error: --gt-scene-flow evaluates the scene flow of --scene-flow; give --scene-flow too", {}),
    (FLOW, SF + ["--odometry", "."], 2,
     "error: --odometry needs the disparities of --scene-flow and the stereo camera of --camera", {}),
    (FLOW, ["--odometry", "."], 2,
     "error: --odometry needs the disparities of --scene-flow and the stereo camera of --camera", {}),
    (ALL, ["--gt-poses", "poses.txt"], 2, "error: --gt-poses evaluates the poses of --odometry; give --odometry too",
     {}),
    (FLOW, ["--fuse", FUSE], 2, "error: --fuse places disparities with the poses of --odometry; give --odometry too",
     {}),
    (ALL, ["--mesh"], 2, "error: --mesh meshes the volume of --fuse; give --fuse too", {}),
    (FLOW, ["--descriptors", "d.txt"], 2, "error: --descriptors describes the clips of --tracks; give --tracks too",
     {}),
    (FLOW, ["--fisher", "cb.fv", "f.txt"], 2, "error: --fisher encodes the clips of --tracks; give --tracks too", {}),
    (FLOW, ["--stabilize", "4", "0.1", "out"], 2,
     "error: --stabilize smooths the models of --global-motion; give --global-motion too", {}),
    (ALL, ["--color-max", "2"], 2, "error: --color-max needs --color", {}),
    # values, checked where they are read
    (FLOW, ODO + ["--fuse", "0.1,0.3,0,0,0,4,4"], 2, "error: --fuse takes eight numbers voxel,trunc,x0,y0,z0,nx,ny,nz "
     "with voxel and trunc > 0, integer sizes >= 1 and at most 2^30 voxels, got 0.1,0.3,0,0,0,4,4", {}),
    (FLOW, ODO + ["--fuse", "0.1,0.3,0,0,0,2048,2048,2048"], 2, "error: --fuse takes eight numbers "
     "voxel,trunc,x0,y0,z0,nx,ny,nz with voxel and trunc > 0, integer sizes >= 1 and at most 2^30 voxels, got "
     "0.1,0.3,0,0,0,2048,2048,2048", {}),
    (FLOW, ["--global-motion", "rigid", "gm.txt"], 2,
     "error: --global-motion takes the model similarity, affine or homography, got rigid", {}),
    (FLOW, ["--tracks", "t.txt", "--fisher", "none.fv", "f.txt"], 2, "error: none.fv: cannot read the codebook", {}),
    (FLOW, ["--tracks", "t.txt", "--fisher", "magic.fv", "f.txt"], 2,
     "error: magic.fv: not a codebook file (OFDISFV1)", {}),
    (FLOW, ["--tracks", "t.txt", "--fisher", "blocks.fv", "f.txt"], 2, "error: blocks.fv: the codebook's blocks are "
     "not the descriptors' (desc_dim 426, blocks 0+30, 30+96, 126+108, 234+96, 330+96)", {}),
    (FLOW, GM + ["--stabilize", "65", "0.1", "out"], 2,
     "error: --stabilize takes a radius 1..64 and a crop 0 <= CROP < 0.5, got 65 0.1", {}),
    (FLOW, GM + ["--stabilize", "4", "0.5", "out"], 2,
     "error: --stabilize takes a radius 1..64 and a crop 0 <= CROP < 0.5, got 4 0.5", {}),
    (STEREO, ["--speckle", "0", "1"], 2,
     "error: --speckle takes a size N >= 1 and a finite difference R >= 0, got 0 1", {}),
    (STEREO, ["--camera", "1,1,0,0,0,0"], 2, "error: --camera takes six finite numbers fx,fy,cx,cy,baseline,doffs "
     "with fx, fy and baseline > 0, got 1,1,0,0,0,0", {}),
    (FLOW, SF + ["--camera", "1,1,0,0"], 2, "error: --camera takes six finite numbers fx,fy,cx,cy,baseline,doffs "
     "with fx, fy and baseline > 0, got 1,1,0,0", {}),
    (ALL, ["--interpolate", "1"], 2, "error: --interpolate takes a time T with 0 < T < 1, got 1", {}),
    (ALL, ["--color", "--color-max", "inf"], 2, "error: --color-max takes a positive finite number, got inf", {}),
    (ALL, ["1", "2", "3"], 2, "error: expected 0, 1 or exactly 20 numbers, got 3", {}),
    (ALL, ["--batch", "0"], 2, "error: expected 0, 1 or exactly 20 numbers, got 0", {}),
    (ALL, ["--batch", "4", "--batch", "0", "2"], 2, "error: expected 0, 1 or exactly 20 numbers, got 1", {}),
    # the rules run in order: the first that fails is the one reported
    (FLOW, ["--warm-start", "--interpolate", "0.5", "--scene-flow", "x"], 2, WARM % "--interpolate", {}),
    (FLOW, ["--interpolate", "2", "--lr-check"], 2, "error: --lr-check, --speckle, --fill and --camera filter stereo "
     "disparities; the flow binaries take none of them", {}),
    (FLOW, ODO + ["--fuse", "x", "--lr-check"], 2, "error: --fuse takes eight numbers voxel,trunc,x0,y0,z0,nx,ny,nz "
     "with voxel and trunc > 0, integer sizes >= 1 and at most 2^30 voxels, got x", {}),
    (FLOW, ["--global-motion", "rigid", "gm.txt", "--descriptors", "d.txt"], 2,
     "error: --global-motion takes the model similarity, affine or homography, got rigid", {}),
    (FLOW, ["--color-max", "0", "--interpolate", "0"], 2,
     "error: --interpolate takes a time T with 0 < T < 1, got 0", {}),
    # the list file and the per-pair inputs
    (ALL, [], 1, None, {}),  # the list file itself does not exist (its own case below)
    (ALL, ["--gt", "none.txt"], 1, "error: cannot read none.txt", {}),
    (ALL, ["--gt", "one.txt"], 2, "error: --gt: one.txt lists 1 ground-truth files for 0 pairs", {}),
    (FLOW, ["--scene-flow", "none.txt"], 1, "error: cannot read none.txt", {}),
    (FLOW, ["--scene-flow", "one.txt"], 2, "error: --scene-flow: one.txt lists 1 files for 0 pairs (2 per pair)", {}),
    (FLOW, SF + ["--gt-scene-flow", "one.txt"], 2,
     "error: --gt-scene-flow: one.txt lists 1 files for 0 pairs (3 per pair)", {}),
    (FLOW, ODO + ["--gt-poses", "none.txt"], 2, "error: cannot read none.txt", {}),
    (FLOW, ODO + ["--gt-poses", "one.txt"], 2, "error: --gt-poses: one.txt lists 1 poses files for 0 clips", {}),
    (FLOW, SF + ["--camera", CAM, "--odometry", "missing"], 2,
     "error: --odometry: cannot write missing/odometry.txt", {}),
    # the list outputs, opened in order: odometry.txt, descriptors, fisher, tracks, stab.txt, global motion
    (FLOW, ODO + ["--tracks", "t.txt", "--descriptors", "missing/d.txt"], 1, "error: cannot write missing/d.txt",
     {"odometry.txt": b""}),
    (FLOW, ["--tracks", "t.txt", "--descriptors", "d.txt", "--fisher", "cb.fv", "missing/f.txt"], 1,
     "error: cannot write missing/f.txt", {"d.txt": DESC_HDR}),
    (FLOW, ["--tracks", "missing/t.txt", "--descriptors", "d.txt", "--fisher", "cb.fv", "f.txt"], 1,
     "error: cannot write missing/t.txt", {"d.txt": DESC_HDR, "f.txt": FISHER_HDR}),
    (FLOW, ["--tracks", "t.txt", "--fisher", "cb.fv", "f.txt"] + GM + ["--stabilize", "4", "0.1", "missing"], 1,
     "error: cannot write missing/stab.txt", {"t.txt": TRACKS_HDR, "f.txt": FISHER_HDR}),
    (FLOW, ODO + ["--tracks", "t.txt", "--global-motion", "affine", "missing/gm.txt", "--stabilize", "4", "0.1",
                  "out"], 1,
     "error: cannot write missing/gm.txt", {"odometry.txt": b"", "t.txt": TRACKS_HDR, "out/stab.txt": b""}),
]

# refusals that read the pairs of a one-pair list (its images are read for their size, or decoded, before any device
# work)
REFUSED_PAIRS = [
    (ALL, "gone.txt", [], 1, "error: cannot read the pair nope1.pgm nope2.pgm " + PAIR, {}),
    (FLOW, "gone.txt", ["--tracks", "t.txt"] + GM, 1, "error: cannot read the pair nope1.pgm nope2.pgm " + PAIR,
     {"t.txt": TRACKS_HDR, "gm.txt": b""}),
    (ALL, "gone.txt", ["--gt", "gt_gone.txt"], 1, "error: cannot read the pair nope1.pgm nope2.pgm " + PAIR, {}),
    (ALL, "pair40.txt", ["--gt", "gt_gone.txt"], 1, "error: g.flo: cannot read the ground-truth file", {}),
    (FLOW, "pair40.txt", ["--scene-flow", "disp40_gone.txt"], 2, "error: gone.pfm: cannot read the ground-truth file",
     {}),
    (FLOW, "pair40.txt", ["--scene-flow", "disp40.txt", "--camera", CAM, "--odometry", ".", "--gt-poses",
                          "poses_gone.txt"], 2, "error: cannot read gone_poses.txt", {}),
    (FLOW, "pair40.txt", ["--scene-flow", "disp40.txt", "--camera", CAM, "--odometry", ".", "--gt-poses",
                          "poses.txt"], 2,
     "error: p0.txt: a KITTI poses file of at least 2 lines of 12 numbers, got 12 numbers", {}),
    (FLOW, "small.txt", ["--tracks", "t.txt", "--descriptors", "d.txt"], 2,
     "error: --descriptors needs frames of at least 32 x 32, a16.pgm is 16 x 16", {}),
    (FLOW, "small.txt", ["--tracks", "t.txt", "--fisher", "cb.fv", "f.txt"], 2,
     "error: --fisher needs frames of at least 32 x 32, a16.pgm is 16 x 16", {}),
    (FLOW, "small.txt", ["--scene-flow", "disp16.txt", "--camera", CAM, "--odometry", ".", "--tracks", "t.txt",
                         "--descriptors", "d.txt"], 2,
     "error: --descriptors needs frames of at least 32 x 32, a16.pgm is 16 x 16", {"odometry.txt": b""}),
    (FLOW, "gone.txt", ["--tracks", "t.txt", "--fisher", "cb.fv", "f.txt"], 1,
     "error: cannot read the pair nope1.pgm nope2.pgm " + PAIR, {}),
]


def _cases(table, with_list):
    out = []
    for row in table:
        exes, rest = row[0], row[1:]
        words = ([rest[0]] if with_list else []) + list(rest[1 if with_list else 0])
        for exe in exes:
            out.append(pytest.param(exe, *rest, id="%s-%s" % (exe, " ".join(words))))
    return out


@pytest.mark.parametrize("exe,args,code,line,left", _cases(REFUSED, False))
def test_refused_before_device_work(bindir, work, exe, args, code, line, left):
    cwd, inputs = work
    lst = "list.txt" if line is not None else "no_such_list.txt"
    r = _run(bindir, exe, [lst] + args, cwd)
    assert r.returncode == code, (r.stdout, r.stderr)
    assert r.stderr == (line if line is not None else "error: cannot read no_such_list.txt") + "\n"
    assert r.stdout == ""
    assert _written(cwd, inputs) == left


@pytest.mark.parametrize("exe,lst,args,code,line,left", _cases(REFUSED_PAIRS, True))
def test_refused_on_the_pairs(bindir, work, exe, lst, args, code, line, left):
    cwd, inputs = work
    r = _run(bindir, exe, [lst] + args, cwd)
    assert r.returncode == code, (r.stdout, r.stderr)
    assert r.stderr == line + "\n"
    assert r.stdout == ""
    assert _written(cwd, inputs) == left


P20 = ["5", "3", "12", "12", "0.05", "0.95", "0", "8", "0.40", "0", "1", "0", "1", "10", "10", "5", "1", "3", "1.6",
       "2"]

# (binaries, arguments after the list file, the files written)
ACCEPTED = [
    (ALL, [], {}),
    (ALL, ["2"], {}),
    (ALL, P20, {}),
    (ALL, ["--batch", "3", "2"], {}),
    (ALL, ["--batch", "0", "--batch", "4"], {}),
    (ALL, ["--batch"], {}),
    (ALL, ["--kitti", "--kitti", "--color", "--color"], {}),
    (ALL, ["--warm-start", "--kitti", "--color", "2"], {}),
    (ALL, ["--bidirectional", "--gt", "empty.txt", "--kitti", "--color", "--color-max", "2", "--interpolate", "0.5"],
     {}),
    (ALL, ["--tracks", "t.txt"], {"t.txt": TRACKS_HDR}),
    (FLOW, ["--tracks", "t.txt", "--descriptors", "d.txt"], {"t.txt": TRACKS_HDR, "d.txt": DESC_HDR}),
    (FLOW, ["--tracks", "t.txt", "--fisher", "cb.fv", "f.txt"], {"t.txt": TRACKS_HDR, "f.txt": FISHER_HDR}),
    (FLOW, ["--tracks", "t.txt", "--descriptors", "d.txt", "--fisher", "cb.fv", "f.txt"],
     {"t.txt": TRACKS_HDR, "d.txt": DESC_HDR, "f.txt": FISHER_HDR}),
    (STEREO, ["--lr-check", "--speckle", "50", "1", "--fill", "--camera", CAM, "--bidirectional"], {}),
    (FLOW, ["--global-motion", "homography", "gm.txt"], {"gm.txt": b""}),
    (FLOW, GM + ["--stabilize", "15", "0.1", "out"], {"gm.txt": b"", "out/stab.txt": b""}),
    (FLOW, SF + ["--gt-scene-flow", "empty.txt", "--camera", CAM], {}),
    (FLOW, ODO + ["--gt-poses", "empty.txt"], {"odometry.txt": b""}),
    (FLOW, ODO + ["--fuse", FUSE, "--mesh"], {"odometry.txt": b""}),
    (FLOW, ["--bidirectional", "--color", "--interpolate", "0.5", "--tracks", "t.txt", "--descriptors", "d.txt",
            "--fisher", "cb.fv", "f.txt", "--global-motion", "affine", "gm.txt", "--stabilize", "4", "0.1", "out",
            "--gt", "empty.txt", "--kitti"] + ODO + ["--gt-poses", "empty.txt", "--fuse", FUSE, "--mesh"],
     {"t.txt": TRACKS_HDR, "d.txt": DESC_HDR, "f.txt": FISHER_HDR, "gm.txt": b"", "out/stab.txt": b"",
      "odometry.txt": b""}),
]


@pytest.mark.parametrize("exe,args,files", [pytest.param(e, a, f, id="%s-%s" % (e, " ".join(a)))
                                            for ex, a, f in ACCEPTED for e in ex])
def test_accepted_on_an_empty_list(bindir, work, exe, args, files):
    cwd, inputs = work
    r = _run(bindir, exe, ["list.txt"] + args, cwd)
    assert (r.returncode, r.stderr) == (0, ""), r.stdout
    assert _written(cwd, inputs) == files


def test_usage(bindir):
    exe = os.path.join(bindir, "run_OF_INT_batch")
    r = subprocess.run([exe], capture_output=True, text=True)
    assert r.returncode == 2
    assert r.stdout == ""
    assert r.stderr == USAGE % exe
