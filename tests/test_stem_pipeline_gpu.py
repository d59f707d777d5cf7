"""The stem's item pipeline (raw bytes double-buffered and converted inside the convolution, two barriers per item, the pooled
rows of an item stored while the next one convolves) bit for bit against tests/golden/stem.npz, at shapes where that pipeline
runs long: CTAs that take many items, the short last band of 352 rows, inputs whose base is not 16-byte aligned (the patch
then arrives by scalar loads; a network input's width is a multiple of 32), 640x640 and an odd number of column tiles.

The golden arrays are of one image each.  A batch holds the golden image among other images; a wider input holds it in its
left columns: with the stem's padding on the left and top only, the first W/4 output columns of a wider image are those of the
image alone (every pool window and conv tap lies inside the first W columns)."""
import importlib.util
import os

import numpy as np
import pytest
import torch

import net_dispatch as nd
import yfv2_engine

_spec = importlib.util.spec_from_file_location(
    "make_golden_stem", os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "make_golden_stem.py"))
mk = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(mk)

SMS = 132                       # H100 SXM
SMEM_PER_SM = 228 * 1024        # shared memory per SM on sm_90
RESERVED_PER_CTA = 1024         # the driver's share of each resident CTA
STATIC_SMEM = 128               # the kernel's own mbarrier, rounded up by ptxas
CTAS_PER_SM = 2                 # __launch_bounds__(256, 2)


def stem_record(n, h, w, u8):
    return nd.host_plan(n, h, w, lambda p: yfv2_engine.plan_launches(p, None, u8, SMS))[0]


@pytest.mark.parametrize("u8", [True, False])
@pytest.mark.parametrize("n,h,w", [(256, 352, 352), (256, 640, 640), (64, 96, 736), (64, 96, 416)])
def test_records_fit_two_ctas_per_sm(n, h, w, u8):
    rec = stem_record(n, h, w, u8)
    assert rec["kernel"] == ("stem_kernel<true>" if u8 else "stem_kernel<false>")
    assert CTAS_PER_SM * (rec["smem"] + STATIC_SMEM + RESERVED_PER_CTA) <= SMEM_PER_SM, rec
    assert rec["grid"][0] == min(rec["items"], CTAS_PER_SM * SMS), rec


def golden_digest(golden_dir, h, w, kind):
    return str(np.load(os.path.join(golden_dir, "stem.npz"))["%dx%d_%s_sha256" % (h, w, kind)])


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["u8", "f32"])
@pytest.mark.parametrize("n,side,at", [(64, 352, (0, 37, 63)), (4, 640, (2,))])
def test_golden_image_inside_a_batch(golden_dir, kind, n, side, at):
    """64 images at 352x352: 2304 items on 264 CTAs, 8 or 9 per CTA, each band set ending in the 3-row band."""
    rec = stem_record(n, side, side, kind == "u8")
    if side == 352:
        assert rec["items"] >= 3 * rec["grid"][0]
    sd_seed, x_seed = mk.seeds(side, side)
    m = mk.make_model(sd_seed)
    x = mk.make_inputs(x_seed + 1, n, side, side)[kind]
    x[list(at)] = mk.make_inputs(x_seed, 1, side, side)[kind]
    out = mk.stem_tap(m, x.cuda())
    want = golden_digest(golden_dir, side, side, kind)
    for i in at:
        assert mk.digest(out[i:i + 1]) == want, i


def unaligned(x):
    """x copied into a CUDA view whose base is one element past an allocation's start (not 16-byte aligned)."""
    buf = torch.empty(x.numel() + 1, dtype=x.dtype, device="cuda")
    v = buf[1:].view(x.shape)
    v.copy_(x)
    assert v.data_ptr() % 16 != 0 and v.is_contiguous()
    return v


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["u8", "f32"])
@pytest.mark.parametrize("aligned", [True, False])
def test_golden_image_in_the_left_columns(golden_dir, kind, aligned):
    """96x416 golden inside 96x736: 184 pooled columns in 5 tiles of 37 (the golden shape runs 3 tiles of 35, 35, 34)."""
    rec = stem_record(3, 96, 736, kind == "u8")
    assert rec["items"] % 3 == 0 and (rec["items"] // 3) % 5 == 0
    sd_seed, x_seed = mk.seeds(96, 416)
    m = mk.make_model(sd_seed)
    x = mk.make_inputs(x_seed + 2, 3, 96, 736)[kind]
    x[1, :, :, :416] = mk.make_inputs(x_seed, 1, 96, 416)[kind][0]
    x = x.cuda() if aligned else unaligned(x)
    out = mk.stem_tap(m, x)
    assert out.shape[-1] == 184
    assert mk.digest(np.ascontiguousarray(out[1:2, :, :, :104])) == golden_digest(golden_dir, 96, 416, kind)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["u8", "f32"])
def test_unaligned_batch_at_352(golden_dir, kind):
    """The scalar-load path over many items per CTA, golden image at both ends of the batch."""
    sd_seed, x_seed = mk.seeds(352, 352)
    m = mk.make_model(sd_seed)
    x = mk.make_inputs(x_seed + 3, 40, 352, 352)[kind]
    x[[0, 39]] = mk.make_inputs(x_seed, 1, 352, 352)[kind]
    out = mk.stem_tap(m, unaligned(x))
    want = golden_digest(golden_dir, 352, 352, kind)
    assert mk.digest(out[0:1]) == want and mk.digest(out[39:40]) == want
