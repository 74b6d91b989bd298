"""Host pre/post-processing (of_dis_b200/preprocess.py) against OpenCV, the library the
reference's main() uses for it (run_dense.cpp:130-178,298-311,407-414).  Skipped where cv2 is
not installed (the GPU box); the device versions of these stages are compared with
preprocess.py in tests/test_gpu_parity.py."""
import numpy as np
import pytest

from of_dis_b200 import preprocess, synth
from test_device_pyramid import GEOMETRIES, geometry_params

cv2 = pytest.importorskip("cv2")


def _pyramid_cases():
    """(ch, size, lv_f, pad): three frame sizes at lv_f 4 and padding 8; then the full-resolution sizes
    and paddings the device pyramids are checked on (tests/test_device_pyramid.py), at lv_f = sc_f up to 7 (the
    4096 x 2048 frames at 6, so that every lv_f from 0 to 7 is reached); then the known limit at level 8 and beyond."""
    cases = [pytest.param(1, (436, 1024), 4, 8, id="1-size0"), pytest.param(3, (121, 203), 4, 8, id="3-size1"),
             pytest.param(1, (64, 96), 4, 8, id="1-size2")]
    for name, g in GEOMETRIES.items():
        lv_f = 6 if name == "deep_sc_f10_4096x2048" else min(geometry_params(g).sc_f, 7)
        cases.append(pytest.param(g["ch"], g["org"], lv_f, g["pad"], id=name))
    assert {c.values[2] for c in cases} == set(range(8))
    cases.append(pytest.param(1, (2048, 1024), 9, 8, id="2048x1024-lv9", marks=pytest.mark.xfail(strict=True, reason=(
        "preprocess.sobel8 sums dy in a different order from cv::Sobel; where those sums round (levels 8 and 9 of "
        "this frame) dy differs by 1-2 ulp, at most 7.6e-6, on 15 and 1 pixels"))))
    return cases


@pytest.mark.parametrize("ch,size,lv_f,pad", _pyramid_cases())
def test_pyramid_gradients_and_paddings_equal_opencv_bitwise(ch, size, lv_f, pad):
    """ConstructImgPyramide (run_dense.cpp:130-178) with cv::resize / cv::Sobel / copyMakeBorder."""
    i0, _, _ = synth.synthetic_pair(size[0], size[1], ch, seed=11)
    img, padw, padh = preprocess.pad_to_multiple(i0, lv_f)
    # run_dense.cpp:299-311
    ref = cv2.copyMakeBorder(i0, padh // 2, padh - padh // 2, padw // 2, padw - padw // 2, cv2.BORDER_REPLICATE)
    assert np.array_equal(img, ref)
    imgs, dxs, dys = preprocess.build_pyramid(img.astype(np.float32), lv_f, pad)
    cur = img.astype(np.float32)
    for lv in range(lv_f + 1):
        if lv > 0:
            cur = cv2.resize(cur, None, fx=0.5, fy=0.5, interpolation=cv2.INTER_LINEAR)
        dx = cv2.Sobel(cur, cv2.CV_32F, 1, 0, ksize=3, scale=1 / 8.0, delta=0, borderType=cv2.BORDER_DEFAULT)
        dy = cv2.Sobel(cur, cv2.CV_32F, 0, 1, ksize=3, scale=1 / 8.0, delta=0, borderType=cv2.BORDER_DEFAULT)
        exp = [cv2.copyMakeBorder(cur, pad, pad, pad, pad, cv2.BORDER_REPLICATE),
               cv2.copyMakeBorder(dx, pad, pad, pad, pad, cv2.BORDER_CONSTANT, value=0),
               cv2.copyMakeBorder(dy, pad, pad, pad, pad, cv2.BORDER_CONSTANT, value=0)]
        for got, e, name in zip((imgs[lv], dxs[lv], dys[lv]), exp, ("image", "dx", "dy")):
            assert got.shape == e.shape
            assert np.array_equal(got.view(np.uint32), e.view(np.uint32)), (lv, name, float(np.abs(got - e).max()))


@pytest.mark.parametrize("nop,lv_l", [(2, 3), (1, 2), (2, 0)])
def test_output_stage_matches_opencv_resize(nop, lv_l):
    """run_dense.cpp:407-414: flow * 2^lv_l, cv::resize(INTER_LINEAR), crop.  cv2 evaluates the
    interpolation in a different order, so the bar here is 1e-5 relative to the flow scale."""
    rng = np.random.default_rng(3)
    h, w = 56, 128
    flow = (rng.standard_normal((h, w, nop)) * 3).astype(np.float32)
    sc = 2 ** lv_l
    got = preprocess.postprocess(flow, lv_l, padw=0, padh=12 if lv_l else 0, width_org=w * sc,
                                 height_org=h * sc - (12 if lv_l else 0))
    ref = flow * np.float32(sc)
    if lv_l:
        ref = cv2.resize(ref, None, fx=sc, fy=sc, interpolation=cv2.INTER_LINEAR).reshape(h * sc, w * sc, nop)
        ref = ref[6:6 + h * sc - 12]
    assert got.shape == ref.shape
    assert float(np.abs(got - ref).max()) <= 1e-5 * sc * 12
