"""CPU side of the NMS parameter space: the C oracle's max_det / max_wh against the numpy restatement, the host-side limits of
yfv2_nms / yfv2_decode_nms (refused before anything is launched, so no GPU is needed), and tests/post_space.py's restatement of
the shared-memory layout."""
import ctypes

import numpy as np
import pytest
import torch

import yfv2  # noqa: F401
import post_space as ps
from oracle import post as opost


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_c_oracle_max_det_and_max_wh_equal_the_numpy_restatement(seed):
    rs = np.random.RandomState(seed)
    d = ps.random_dets(300 + seed, 2, 400, classes=6, side=352.0)
    d[1, ::4, 2] *= 30.0                                       # wide boxes: classes overlap after small offsets
    for max_det in (1, 7, 64, 65, 300, 1000):
        for max_wh in (4096.0, 1024.0, 100.0, 0.0):
            ct, it = float(rs.choice([0.001, 0.3])), float(rs.choice([0.3, 0.45, 0.5]))
            a, ia = opost.nms(torch.from_numpy(d), ct, it, return_indices=True, max_det=max_det, max_wh=max_wh)
            b, ib = opost.nms(torch.from_numpy(d), ct, it, return_indices=True, max_det=max_det, max_wh=max_wh, impl="numpy")
            for i in range(2):
                assert np.array_equal(a[i].numpy(), b[i].numpy()), (max_det, max_wh, i)
                assert np.array_equal(ia[i], ib[i]), (max_det, max_wh, i)
                assert a[i].shape[0] <= max_det
    # the defaults are the reference's (cap 300, offset 4096)
    x = ps.random_dets(310, 1, 1815, side=352.0)
    r0, _ = opost.nms_image_c(x[0], 0.001, 0.45)
    r1, _ = opost.nms_image_c(x[0], 0.001, 0.45, max_det=300, max_wh=4096.0)
    assert r0.shape[0] == 300 and np.array_equal(r0, r1)


def test_nms_limits_are_refused_before_any_launch():
    import yfv2_engine
    lib = yfv2_engine.lib()
    fake = ctypes.c_void_p(256)                                # never dereferenced: every case fails its host-side check

    def nms(M, max_det):
        return lib.yfv2_nms(fake, 1, M, 80, ctypes.c_float(0.3), ctypes.c_double(0.45), None, 0, max_det, ctypes.c_float(4096.0),
                            fake, fake, fake, None, None)
    assert nms(1815, 0) == -1 and b"bad arguments" in lib.yfv2_last_error()
    assert nms(1815, 4097) == -1
    assert nms(ps.MAX_CAND + 1, 300) == -3 and b"8192" in lib.yfv2_last_error()
    assert ps.nms_smem_bytes(ps.MAX_CAND, 801) <= ps.SMEM_CAP < ps.nms_smem_bytes(ps.MAX_CAND, 802)
    assert nms(ps.MAX_CAND, 802) == -3 and b"shared memory" in lib.yfv2_last_error()
    assert ps.largest_cap(6000) == 2774
    assert nms(6000, 2775) == -3 and b"shared memory" in lib.yfv2_last_error()

    six = (ctypes.c_void_p * 6)(*([256] * 6))
    anchors = (ctypes.c_double * 32)(*range(1, 33))

    def fused(H, W, A, C, max_det):
        return lib.yfv2_decode_nms(six, 1, H, W, A, C, anchors, ctypes.c_float(0.3), ctypes.c_double(0.45), None, 0, max_det,
                                   ctypes.c_float(4096.0), fake, fake, fake, None, None)
    assert fused(352, 352, 3, 80, 0) == -1 and fused(352, 352, 3, 80, 4097) == -1
    assert fused(1024, 1024, 3, 80, 300) == -3 and b"8192" in lib.yfv2_last_error()   # M = 15360
    cap = ps.largest_cap(8160)                                 # A = 8 at 384 x 544: M = 8160, thread-per-cell (no staging)
    assert fused(384, 544, 8, 20, cap + 1) == -3 and b"shared memory" in lib.yfv2_last_error()


def test_shared_memory_restatement():
    """post_space.nms_smem_bytes / lists_fit restate k_post.cu; spot values pin the arithmetic the GPU tests build on."""
    assert ps.pow2_at_least(1) == 64 and ps.pow2_at_least(65) == 128 and ps.pow2_at_least(8192) == 8192
    assert ps.largest_cap(1815) == 4096 and ps.largest_cap(8192) == 801
    # lists need 8 (MCp - M) >= 4 max_det + 512 and max_det >= 64
    assert ps.lists_fit(1815, 338) and not ps.lists_fit(1815, 339) and not ps.lists_fit(1815, 63)
    assert not ps.lists_fit(2048, 64) and ps.lists_fit(6000, ps.largest_cap(6000))
    assert [ps.sort_size(c) for c in (0, 64, 65, 256, 257, 2048, 2049, 8192)] == [64, 64, 128, 256, 512, 2048, 4096, 8192]
