"""The batch command's --confidence grammar on CPU: each refusal before any device work, with its exit code and its
whole stderr line, on every binary, and the empty list it accepts."""
import subprocess

import pytest

from of_dis_b200 import build

ALL = ["run_OF_INT", "run_OF_RGB", "run_DE_INT", "run_DE_RGB"]


@pytest.fixture(scope="module")
def bindir():
    return build.build_host()


@pytest.mark.parametrize("binary", ALL)
@pytest.mark.parametrize("args,line", [
    (["--confidence"], "error: --confidence takes one window radius"),
    (["--confidence", "2", "--confidence", "3"], "error: --confidence takes one window radius"),
    (["--confidence", "0"], "error: --confidence takes a radius 1..7, got 0"),
    (["--confidence", "8"], "error: --confidence takes a radius 1..7, got 8"),
    (["--confidence", "2x"], "error: --confidence takes a radius 1..7, got 2x"),
    (["--confidence", "-1"], "error: --confidence takes a radius 1..7, got -1"),
    (["--warm-start", "--confidence", "2"], "error: --warm-start runs one pair per launch; it takes no --confidence"),
    (["--confidence", "2", "--color-max", "3"], "error: --color-max needs --color"),
])
def test_refusals(binary, args, line, bindir, tmp_path):
    (tmp_path / "list.txt").write_text("")
    r = subprocess.run([str(bindir) + "/" + binary + "_batch", "list.txt"] + args, capture_output=True, text=True,
                       cwd=str(tmp_path))
    assert r.returncode == 2 and r.stderr == line + "\n", (r.returncode, r.stderr)
    assert sorted(q.name for q in tmp_path.iterdir()) == ["list.txt"]


@pytest.mark.parametrize("binary", ALL)
@pytest.mark.parametrize("radius", ["1", "7"])
def test_accepted_on_an_empty_list(binary, radius, bindir, tmp_path):
    (tmp_path / "list.txt").write_text("")
    r = subprocess.run([str(bindir) + "/" + binary + "_batch", "list.txt", "--confidence", radius, "--bidirectional"],
                       capture_output=True, text=True, cwd=str(tmp_path))
    assert r.returncode == 0 and r.stderr == "", (r.returncode, r.stderr)
    assert "CONF" not in r.stdout
    assert sorted(q.name for q in tmp_path.iterdir()) == ["list.txt"]
