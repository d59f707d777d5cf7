"""The forward, training and augmentation kernels at SM counts and persistent grid sizes other than this device's, bit for bit.

The SM count decides the band height of the block launches, the grids of the stem, FPN and heads, the wgrad pixel chunks and the
grid caps of the copies and the augmentation kernels; the persistent launches take one CTA per item up to what occupancy allows.
Several kernels carry state from one item to the next (the stride-1 walk stages the next item's rows, the stem prefetches the next
item, the staged heads copy ahead into the next item, the chain overlaps the next block's weights with its last image), so their
result could depend on the sequence of items each CTA walks.  yfv2_engine.simulated_dispatch runs the same plan as another GPU
would dispatch it; every tensor of the forward must equal, bit for bit, the forward at this device's own count, and the profiler
trace must show the simulated grids.  A few cases are also checked launch by launch against the fp64 oracle, a reference that does
not depend on the run at this device's count.  -s prints, per case, the launches whose geometry or grid differs.

tests/test_dispatch_counts_gpu.py runs this module in a process of its own: after a CUDA activity session, a later session in the
same process that starts a few minutes on loses the records of its first kernels, which tests/test_forward_fp64_gpu.py's trace of
a forward would trip over."""
import time

import pytest
import torch

import yfv2  # noqa: F401
import yfv2_engine as eng
import net_dispatch as nd
from test_forward_fp64_gpu import (BOUND, TRACE_MARGIN_S, io_taps, nerr, reference, setup, traced_launches,  # noqa: F401
                                   tracer_ready)

pytestmark = pytest.mark.gpu

# name -> (N, H, W); every one reaches a different mix of band geometries when the SM count is small
SHAPES = {"1x32x32": (1, 32, 32), "2x64x96": (2, 64, 96), "1x128x128": (1, 128, 128), "4x128x128": (4, 128, 128),
          "1x352x352": (1, 352, 352), "8x352x352": (8, 352, 352), "1x640x32": (1, 640, 32), "1x1280x128": (1, 1280, 128),
          "2x256x1280": (2, 256, 1280)}
SEED = {name: 3000 + 10 * i for i, name in enumerate(SHAPES)}
SM_COUNTS = (1, 2, 3, 7, 16, 33, 78, 114, 148, 264, 1024)      # MIG slices up to twice a B200
CTA_CAPS = (1, 2, 3, 5)
ORACLE_CASES = [(name, sms) for name in ("2x64x96", "1x128x128", "1x352x352") for sms in (1, 16)]
GATHER_IDS = range(23)                                          # yfv2_debug_gather: stem, 16 blocks, S2, S3, mid-head scratch


def device_sms():
    return torch.cuda.get_device_properties(0).multi_processor_count if torch.cuda.is_available() else 132


def changed(a, b):
    """the launches of record list a whose kernel, band geometry or fixed grid differs from b's (same stages)"""
    assert [L.names for L in a] == [L.names for L in b]
    return [L for L, B in zip(a, b) if (L.kernel, L.R, L.bands, L.grid) != (B.kernel, B.R, B.bands, B.grid)]


def sim_cases(base_sms):
    """(shape, sms) pairs whose forward launches differ, on the host records alone, from those at base_sms SMs"""
    return [(name, sms) for name, s in SHAPES.items() for sms in SM_COUNTS
            if sms != base_sms and changed(nd.launches(*s, sms=sms), nd.launches(*s, sms=base_sms))]


def cta_caps(name, sms):
    """CTA caps {1, 2, 3, 5, items - 1, items} over the persistent launches of the shape at sms SMs"""
    items = {L.items for L in nd.launches(*SHAPES[name], sms=sms) if L.grid is None}
    return sorted(set(CTA_CAPS) | {i for n in items for i in (n - 1, n) if i > 0})


SIM_CASES = sim_cases(device_sms())
# the caps at this device's count, and at 16 SMs, where the stride-1 walks of 8 x 352 x 352 end each image on a two-row partial
# band: only a CTA that walks consecutive bands stages there a next item whose rows miss the ring by one (a + a2 = 2G + 3)
CTA_CASES = [(name, sms, c) for sms in (0, 16) for name in SHAPES for c in cta_caps(name, sms or device_sms())
             if sms == 0 or name == "8x352x352"]


# ---- forward ------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def runs():
    """(name, u8) -> (plan, input, every tensor of the forward at this device's own dispatch), built once per module"""
    cache = {}

    def get(name, u8):
        if (name, u8) not in cache:
            n, h, w = SHAPES[name]
            m, _, x, _ = setup(name, (n, h, w, 3, 80, None), SEED[name])
            preds = m(x)
            plan = next(iter(m._plans.values()))
            if u8:
                x = (x * 255).to(torch.uint8)
            cache[(name, u8)] = (m, plan, x, run(plan, x, preds))
        return cache[(name, u8)][1:]
    return get


def run(plan, x, preds):
    """one forward from a cleared workspace and NaN head tensors; returns the 23 gathered tensors and the six head tensors"""
    plan.workspace.fill_(255)
    eng._check(eng.lib().yfv2_plan_invalidate_workspace(plan._h), "plan_invalidate_workspace")   # the forward zeroes it again
    for p in preds:
        p.fill_(float("nan"))
    plan.forward(x, preds)
    return [plan.debug_gather(i) for i in GATHER_IDS] + [p.clone() for p in preds]


def traced_run(plan, x, tmp_path):
    """run() inside a CUDA activity trace: (tensors, traced launches of the forward)"""
    preds = plan.alloc_preds()
    box = []
    got = traced_launches(lambda: box.append(run(plan, x, preds)), tmp_path / "forward.json")
    return box[0], got


def check_trace(model, got, ctas, sms):
    """kernel names and exact grids of the traced forward against its records"""
    assert [k for k, _, _, _ in got] == [L.kernel for L in model], ([k for k, *_ in got], [L.kernel for L in model])
    for L, (_, grid, _, _) in zip(model, got):
        if L.grid is not None:
            assert grid == L.grid, (L.names, grid, L.grid)
        elif ctas:
            assert grid == (min(L.items, ctas), 1, 1), (L.names, grid, L.items, ctas)
        else:                             # occupancy-sized: one to eight 256-thread CTAs per SM, at most one per item
            assert min(L.items, sms) <= grid[0] <= min(L.items, 8 * sms) and grid[1:] == (1, 1), (L.names, grid, L.items, sms)


def check_equal(name, want, got):
    bad = [i for i, (a, b) in enumerate(zip(want, got)) if not torch.equal(a, b)]
    assert not bad, "%s: tensors %s differ (0-22: debug_gather ids, 23-28: head tensors)" % (name, bad)


def describe(rows):
    return "; ".join("%s %s" % (nm, d) for nm, d in rows) or "nothing"


@pytest.mark.parametrize("u8", [False, True], ids=["f32", "u8"])
@pytest.mark.parametrize("name,sms", SIM_CASES, ids=["%s-%dsm" % c for c in SIM_CASES])
def test_forward_at_other_sm_counts_is_bit_identical(name, sms, u8, runs, tmp_path, tracer_ready):
    plan, x, want = runs(name, u8)
    own, own_sms = nd.plan_launches(plan, u8), device_sms()
    _, own_trace = traced_run(plan, x, tmp_path)
    with eng.simulated_dispatch(sms):
        model = nd.plan_launches(plan, u8)
        got, trace = traced_run(plan, x, tmp_path)
    check_trace(model, trace, 0, sms)
    rows = [(L.names[0], "R=%d bands=%d -> R=%d bands=%d" % (B.R, B.bands, L.R, L.bands)) for L, B in zip(model, own)
            if (L.R, L.bands) != (B.R, B.bands)]
    rows += [(L.names[0], "grid %s -> %s" % (a[1], b[1])) for L, a, b in zip(model, own_trace, trace) if a[1] != b[1]]
    print("\n%s %s at %d SMs (device %d): %s" % (name, "u8" if u8 else "f32", sms, own_sms, describe(rows)))
    assert rows, "the simulated dispatch changed no launch"
    check_equal(name, want, got)


@pytest.mark.parametrize("name,sms,ctas", CTA_CASES, ids=["%s-%s-%dctas" % (n, "%dsm" % s if s else "own", c) for n, s, c in CTA_CASES])
def test_forward_at_other_persistent_grids_is_bit_identical(name, sms, ctas, runs, tmp_path, tracer_ready):
    plan, x, want = runs(name, False)
    with eng.simulated_dispatch(sms, ctas):
        model = nd.plan_launches(plan)
        got, trace = traced_run(plan, x, tmp_path)
    check_trace(model, trace, ctas, sms or device_sms())
    print("\n%s at %d SMs, at most %d CTAs: %s" % (name, sms or device_sms(), ctas, describe(
        [(L.names[0], "%d items on %d CTAs" % (L.items, g[1][0])) for L, g in zip(model, trace) if L.grid is None])))
    check_equal(name, want, got)


@pytest.mark.parametrize("name,sms", ORACLE_CASES, ids=["%s-%dsm" % c for c in ORACLE_CASES])
def test_every_launch_at_other_sm_counts_against_fp64(name, sms):
    """each launch, fed what the GPU consumed, against the fp64 oracle at the bound of tests/test_forward_fp64_gpu.py"""
    n, h, w = SHAPES[name]
    m, sd, x, imgs = setup(name, (n, h, w, 3, 80, None), SEED[name])
    sd64 = {k: v.double() if v.is_floating_point() else v for k, v in sd.items()}
    preds = m(x)
    plan = next(iter(m._plans.values()))
    idx = torch.tensor(imgs, device="cuda")
    rows = []
    with eng.simulated_dispatch(sms):
        for L in nd.plan_launches(plan):
            tin, tout = io_taps(L)
            ins = [plan.debug_gather(t)[idx].double().cpu() for t in tin] if tin else [x[idx].double().cpu()]
            plan.forward_range(x, preds, L.first, L.last)
            if tout == "preds":
                lv = int(L.names[0][5]) - 2
                got = [p[idx].double().cpu() for p in preds[3 * lv:3 * lv + 3]]
            else:
                got = [plan.debug_gather(t)[idx].double().cpu() for t in tout]
            rows.append((L, max(nerr(g, r) for g, r in zip(got, reference(L, sd64, ins)))))
    print("\n%s at %d SMs" % (name, sms))
    for L, e in rows:
        print("  %-12s %-24s R=%-3d bands=%-3d %.3e" % (L.names[0], L.kernel, L.R, L.bands, e))
    bad = [(L.names[0], e) for L, e in rows if not e <= BOUND]
    assert not bad, bad


# ---- training -----------------------------------------------------------------------------------------------------------------
def kernel_trace(fn, path, names):
    """(kernel, grid) of every kernel fn() ran whose demangled name is one of `names` (or starts with one ending in "<"), in start
    order (graph launches included)"""
    import json
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        time.sleep(TRACE_MARGIN_S)                 # records at the session's edges can be lost (test_forward_fp64_gpu.py)
        fn()
        torch.cuda.synchronize()
        time.sleep(TRACE_MARGIN_S)
    prof.export_chrome_trace(str(path))
    out = []
    for e in sorted((e for e in json.load(open(path))["traceEvents"] if e.get("cat") == "kernel"), key=lambda e: e["ts"]):
        s = e["name"].replace(" ", "")
        k = [k for k in names if ("::" + k if k.endswith("<") else "::%s(" % k) in s]
        if k:
            out.append((k[0], tuple(e["args"]["grid"])))
    return out


def wgrad(rs):
    return [(r["kernel"], r["pchunk"], r["chunks"], r["partial"], r["grid"]) for r in rs if r["kernel"].startswith("wgrad")]


def op_sm_counts(case):
    """SM counts at which the conv1x1_bwd weight gradient of a test_train_ops_space_gpu.PW case changes its pixel chunking"""
    n, k, m, h, w, bias, _ = case
    recs = lambda s: wgrad(eng.op_launches("conv1x1_bwd", [1 << 20] * 5 + [(1 << 20) if bias else None], [n, k, m, h * w], s))
    return [s for s in SM_COUNTS if recs(s) != recs(device_sms())]


def _op_cases():
    import test_train_ops_space_gpu as sp
    return [(c, s) for c in sp.PW for s in op_sm_counts(c)]


OP_CASES = _op_cases()


@pytest.mark.parametrize("case,sms", OP_CASES, ids=["N%d_K%d_M%d_%dx%d-%dsm" % (c[:5] + (s,)) for c, s in OP_CASES])
def test_conv1x1_bwd_at_other_sm_counts(case, sms, tmp_path):
    """dx bit-identical to this device's count (its GEMM does not depend on it), dw and dbias within the fp64 bound"""
    from test_train_fp64_gpu import TAU, nerr as tnerr, ref_op
    from test_train_ops_space_gpu import buf, empty, op
    n, k, m, h, w, bias, off = case
    g = torch.Generator(device="cuda").manual_seed(hash(case) % 2 ** 31)
    x, wt = buf((n, k, h, w), off, g), buf((m, k, 1, 1), off, g, k ** -0.5)
    dy = buf((n, m, h, w), off, g)

    def bwd():
        dx, dw, db = empty((n, k, h, w), off), empty((m, k, 1, 1), off), empty((m,), off) if bias else None
        op("conv1x1_bwd", [x, wt, dy, dx, dw, db, n, k, m, h * w])
        return dx, dw, db
    dx0, _, _ = bwd()
    args = lambda p: [p(x), p(wt), p(dy), p(dx0), p(dx0), p(dx0) if bias else None]
    with eng.simulated_dispatch(sms):
        recs = eng.op_launches("conv1x1_bwd", args(lambda t: t.data_ptr()), [n, k, m, h * w])
        box = []
        trace = kernel_trace(lambda: box.append(bwd()), tmp_path / "op.json", {r["kernel"] for r in recs if r["kernel"] != "memset"})
    dx, dw, db = box[0]
    assert trace == [(r["kernel"], r["grid"]) for r in recs if r["kernel"] != "memset"], trace
    R = ref_op("pw", {}, {"x": x.double(), "dy": dy.double(), "w": wt.double(), "bias": None})
    errs = {"dw": tnerr(dw, *R["dw"])}
    if bias:
        errs["dbias"] = tnerr(db, dy.double().sum((0, 2, 3)), dy.double().abs().sum((0, 2, 3)))
    print("\n  %s at %d SMs: wgrad %s, %s" % (case, sms, wgrad(recs), errs))
    assert torch.equal(dx, dx0)
    assert all(e <= TAU for e in errs.values()), errs


TRAIN_CASE = "2x640x352"        # its wgrad slices move at one SM, its chan_copy and axpy grids at one SM and at 264


def test_trainer_recaptures_at_other_sm_counts(tmp_path):
    """One trainer stepped at 1 SM, at 264 and back at this device's count: each step's traced grids are its own records (a graph
    captured under another dispatch would replay the old grids), and every op is within the fp64 bound of
    tests/test_train_fp64_gpu.py."""
    import test_train_fp64_gpu as tf
    n, h, w, _, _ = tf.CASES[TRAIN_CASE]
    m = None
    for sms in (1, 264, 0):
        with eng.simulated_dispatch(sms):
            step = tf.run_step(TRAIN_CASE, m) if m is None else None        # builds the model and its trainer
            m = step[0] if step else m
            tr = m._trainer_for(torch.empty((n, 3, h, w), device="cuda"))
            recs = [r for r in eng.trainer_launches(tr._h, tr.workspace.data_ptr()) if r["kernel"] != "memset"]
            box = []
            trace = kernel_trace(lambda: box.append(tf.run_step(TRAIN_CASE, m)), tmp_path / "step.json", {r["kernel"] for r in recs})
            ck = tf.check_case(TRAIN_CASE, step=box[0])[0]
        assert trace == [(r["kernel"], r["grid"]) for r in recs], (sms, len(trace), len(recs))
        worst = max(ck.rows.values())
        print("\n  %s at %s SMs: %d launches traced as recorded, worst op error %.2e" % (TRAIN_CASE, sms or device_sms(), len(trace), worst))
        assert not ck.exact_fail, ck.exact_fail
        assert worst <= tf.TAU, sorted((s, e) for s, e in ck.rows.items() if not e <= tf.TAU)[:10]


# ---- augmentation -------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("sms", [1, 2])
def test_augmentation_at_few_sms(sms, tmp_path):
    """256 x 256 images: 4096 16-byte units per plane, so each thread of the 4 x sms-CTA grids loops over several"""
    import numpy as np
    from oracle import aug as oaug
    from test_aug_blur_gpu import draws, oracle
    N, H, W = 4, 256, 256
    rs = np.random.RandomState(sms)
    x = rs.randint(0, 256, (N, 3, H, W)).astype(np.uint8)
    a, b, rw, rh, r, blur = draws(N, H, W, 7 + sms, every=2)
    luts = eng.hsv_luts(r)
    d = torch.from_numpy(x).cuda()
    names = {"contrast_brightness_kernel", "aug_pixel_kernel<"}
    with eng.simulated_dispatch(sms):
        box = []
        trace = kernel_trace(lambda: box.extend([eng.contrast_and_brightness(d, a, b), eng.augment_batch(d, a, b, luts=luts),
                                                 eng.augment_batch(d, a, b, luts=luts, blur=blur)]), tmp_path / "aug.json", names)
    assert [g[0] for _, g in trace] == [4 * sms] * 3 and len(trace) == 3, trace      # the pixel kernels' grid cap, 4 x SMs
    cb, pix, blurred = (t.cpu().numpy() for t in box)
    for n in range(N):
        src = x[n].transpose(1, 2, 0)
        assert np.array_equal(cb[n], oaug.contrast_and_brightness(x[n], a[n], b[n])), n
        assert np.array_equal(pix[n].transpose(1, 2, 0), oracle(src, 5, a[n], b[n], rw[n], rh[n], r[n], blur[n])), n
        assert np.array_equal(blurred[n].transpose(1, 2, 0), oracle(src, 13, a[n], b[n], rw[n], rh[n], r[n], blur[n])), n
