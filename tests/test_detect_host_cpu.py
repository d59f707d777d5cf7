"""CPU checks of yfv2_detect_u8_host's argument validation: a request the fused decode+NMS cannot run must be refused with the
NMS's own error before anything is enqueued (plans are host-only objects, so no device is needed to see the refusal; without one,
a call that got as far as its host->device copy reports a CUDA error instead)."""
import ctypes

import pytest

import yfv2  # noqa: F401
import post_space as ps

YFV2_EINVAL, YFV2_ECUDA, YFV2_EUNSUPPORTED = -1, -2, -3


@pytest.fixture
def plan():
    import yfv2_engine
    lib = yfv2_engine.lib()
    made = []

    def make(N, H, W, A=3, C=80):
        h = ctypes.c_void_p()
        assert lib.yfv2_plan_create(ctypes.byref(h), 0, N, H, W, A, C, 0) == 0, lib.yfv2_last_error()
        made.append(h)
        return h
    yield make
    for h in made:
        assert lib.yfv2_plan_destroy(h) == 0


def detect(plan_h, max_det, A=3):
    """The whole step with dummy (never dereferenced) pointers for every buffer."""
    import yfv2_engine
    lib = yfv2_engine.lib()
    dummy = ctypes.c_void_p(4096)
    anchors = (ctypes.c_double * (4 * A))(*([10.0] * (4 * A)))
    rc = lib.yfv2_detect_u8_host(plan_h, dummy, dummy, anchors, ctypes.c_float(0.001), ctypes.c_double(0.4), max_det, dummy, dummy,
                                 dummy, None)
    return rc, lib.yfv2_last_error().decode()


def side_m(side, A=3):
    return A * ((side // 16) ** 2 + (side // 32) ** 2)


@pytest.mark.parametrize("side,max_det,rc_want,msg", [
    (1024, 300, YFV2_EUNSUPPORTED, "nms: M=15360 candidates per image exceeds 8192"),   # plan_create accepts 1024^2
    (352, 4097, YFV2_EINVAL, "nms: bad arguments"),
    (352, 5000, YFV2_EINVAL, "nms: bad arguments"),
    (736, ps.largest_cap(side_m(736)) + 1, YFV2_EUNSUPPORTED, "decode_nms: "),          # the smallest cap whose state does not fit
    (736, 4096, YFV2_EUNSUPPORTED, "decode_nms: "),                                      # the largest cap the 4096 rule lets through
], ids=["1024x1024", "max_det_4097", "max_det_5000", "smem_first_over", "smem_max_det_4096"])
def test_refused_with_the_nms_error_before_the_copy(plan, side, max_det, rc_want, msg):
    assert side_m(736) == 7935 and ps.largest_cap(7935) < 4096
    rc, err = detect(plan(2, side, side), max_det)
    assert rc == rc_want and err.startswith(msg), (rc, err)
    if msg == "decode_nms: ":
        assert err.endswith("bytes of shared memory needed"), err


def test_largest_fitting_cap_gets_past_the_checks(plan):
    """At the largest cap that fits, the checks pass and the call goes on to its copy: a CUDA error on a machine without a
    device, success with one (not exercised here: the pointers are dummies)."""
    import torch
    if torch.cuda.is_available():
        pytest.skip("the dummy pointers would be dereferenced by a real copy")
    rc, err = detect(plan(1, 736, 736), ps.largest_cap(7935))
    assert rc == YFV2_ECUDA, (rc, err)


def test_bad_max_det_and_null_pointers(plan):
    h = plan(1, 64, 64)
    for md in (0, -1):
        assert detect(h, md)[0] == YFV2_EINVAL
    import yfv2_engine
    lib = yfv2_engine.lib()
    anchors = (ctypes.c_double * 12)(*([10.0] * 12))
    d = ctypes.c_void_p(4096)
    assert lib.yfv2_detect_u8_host(h, None, d, anchors, ctypes.c_float(0.3), ctypes.c_double(0.4), 10, d, d, d, None) == YFV2_EINVAL
    assert lib.yfv2_detect_u8_host(h, d, d, None, ctypes.c_float(0.3), ctypes.c_double(0.4), 10, d, d, d, None) == YFV2_EINVAL
    assert lib.yfv2_detect_u8_host(h, d, d, anchors, ctypes.c_float(0.3), ctypes.c_double(0.4), 10, d, d, None, None) == YFV2_EINVAL
