"""The batch command's --mono-odometry and --intrinsics grammar on CPU: each refusal before any device work, with its
exit code and its whole stderr line, on every binary, and --gt-poses's refusal without either odometry unchanged."""
import subprocess

import pytest

from of_dis_b200 import build

ALL = ["run_OF_INT", "run_OF_RGB", "run_DE_INT", "run_DE_RGB"]
FLOW = ALL[:2]
STEREO = ALL[2:]
K = "721.5,721.5,609.6,172.9"


@pytest.fixture(scope="module")
def bindir():
    return build.build_host()


def run(bindir, binary, args, tmp_path):
    (tmp_path / "list.txt").write_text("")
    return subprocess.run([str(bindir) + "/" + binary + "_batch", "list.txt"] + args, capture_output=True, text=True,
                          cwd=str(tmp_path))


def check(r, line, tmp_path):
    assert r.returncode == 2 and r.stderr == "error: " + line + "\n", (r.returncode, r.stderr)
    assert sorted(q.name for q in tmp_path.iterdir()) == ["list.txt"]


@pytest.mark.parametrize("binary", STEREO)
@pytest.mark.parametrize("args,line", [
    (["--mono-odometry", ".", "--intrinsics", K],
     "--mono-odometry fits the camera's motion from flows; the stereo binaries take no --mono-odometry"),
    (["--mono-odometry", "."],
     "--mono-odometry fits the camera's motion from flows; the stereo binaries take no --mono-odometry"),
    (["--intrinsics", K],
     "--intrinsics calibrates the camera of --mono-odometry; the stereo binaries take no --intrinsics"),
])
def test_stereo_binaries_refuse(binary, args, line, bindir, tmp_path):
    check(run(bindir, binary, args, tmp_path), line, tmp_path)


@pytest.mark.parametrize("binary", FLOW)
@pytest.mark.parametrize("args,line", [
    (["--warm-start", "--mono-odometry", ".", "--intrinsics", K],
     "--warm-start runs one pair per launch; it takes no --mono-odometry"),
    (["--mono-odometry", "."], "--mono-odometry needs the camera intrinsics of --intrinsics"),
    (["--intrinsics", K], "--intrinsics calibrates the camera of --mono-odometry; give --mono-odometry too"),
    (["--mono-odometry", "missing", "--intrinsics", K], "--mono-odometry: cannot write missing/monodometry.txt"),
    (["--mono-odometry"], "--mono-odometry takes one output directory"),
    (["--mono-odometry", ".", "--intrinsics"], "--intrinsics takes fx,fy,cx,cy"),
] + [(["--mono-odometry", ".", "--intrinsics", bad],
      "--intrinsics takes four finite numbers fx,fy,cx,cy with fx and fy > 0, got " + bad)
     for bad in ("721.5,721.5,609.6", "721.5,721.5,609.6,172.9,1", "0,721.5,609.6,172.9", "721.5,-1,609.6,172.9",
                 "721.5,721.5,inf,172.9", "721.5,721.5,609.6,nan", "a,b,c,d", "721.5,721.5,609.6,172.9x", "")])
def test_flow_binaries_refuse(binary, args, line, bindir, tmp_path):
    check(run(bindir, binary, args, tmp_path), line, tmp_path)


@pytest.mark.parametrize("binary", ALL)
def test_gt_poses_refusal_is_unchanged(binary, bindir, tmp_path):
    check(run(bindir, binary, ["--gt-poses", "poses.txt"], tmp_path),
          "--gt-poses evaluates the poses of --odometry; give --odometry too", tmp_path)


@pytest.mark.parametrize("binary", FLOW)
def test_accepted_on_an_empty_list(binary, bindir, tmp_path):
    (tmp_path / "out").mkdir()
    r = run(bindir, binary, ["--mono-odometry", "out", "--intrinsics", K, "--bidirectional"], tmp_path)
    assert r.returncode == 0 and r.stderr == "", (r.returncode, r.stderr)
    assert (tmp_path / "out" / "monodometry.txt").read_text() == ""
