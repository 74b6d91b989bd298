"""Consecutive frames (CPU side): the synthetic clip generator, and the batch front-end's argument handling on a
list whose pairs form a chain."""
import os
import subprocess

import numpy as np
import pytest

from of_dis_b200 import api, build, synth


@pytest.mark.parametrize("h,w,ch,seed,amp,stereo", [(40, 60, 1, 3, 6.0, False), (33, 47, 3, 5, 3.0, True)])
def test_synthetic_sequence_starts_with_the_synthetic_pair(h, w, ch, seed, amp, stereo):
    seq = synth.synthetic_sequence(4, h, w, ch, seed=seed, amp=amp, stereo=stereo)
    i0, i1, _ = synth.synthetic_pair(h, w, ch, seed=seed, amp=amp, stereo=stereo)
    assert seq.dtype == np.uint8 and seq.shape == (4,) + i0.shape
    assert np.array_equal(seq[0], i0) and np.array_equal(seq[1], i1)
    for t in range(3):
        assert (seq[t] != seq[t + 1]).any(), t


def test_sequence_upload_is_exported():
    assert "ofdis_upload_sequence_u8" in api.EXPORTS


def test_batch_front_end_errors_on_a_chained_list_of_missing_files(tmp_path):
    exe = os.path.join(build.build_host(), "run_OF_INT_batch")
    lst = tmp_path / "list.txt"
    lst.write_text("".join("/nonexistent/f%d.png /nonexistent/f%d.png %s\n" % (k, k + 1, tmp_path / ("o%d.flo" % k))
                           for k in range(4)))
    assert subprocess.run([exe], capture_output=True).returncode == 2
    r = subprocess.run([exe, str(lst), "--batch", "2", "2"], capture_output=True)
    assert r.returncode == 1 and b"cannot read the pair" in r.stderr
    r = subprocess.run([exe, str(lst), "1", "2", "3"], capture_output=True)
    assert r.returncode == 2 and b"20" in r.stderr
