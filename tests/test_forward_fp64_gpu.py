"""Every kernel launch of the forward, one at a time, against an fp64 restatement of the same operation (oracle/net.py with
float64 weights), at band geometries picked with the dispatch model (tests/net_dispatch.py) so that together the cases reach
every (launch site, variant) cell: one-row, multi-row and partial-last bands, chains, whole-image kernels, both head kernels.

Each launch is fed the input the GPU actually consumed (the taps gathered right before it runs, sliced on the device to the
checked images and promoted to float64), so error does not compound across launches and one tight bound holds for all of them.
The metric, per checked image and output tensor, is max|gpu - ref64| / max(max|ref64|, 1e-3); -s prints the worst per launch.
Measured on an H100 80GB HBM3 (132 SMs, 700 W power limit), the worst over all cases is 3.6e-6 for a single launch (fpn.S2,
a 288-deep contraction; every block launch stays under 2.3e-6) and 3.0e-6 for the head tensors end to end.  The bounds below
sit 3.3x and 5x above those.  Dropping one of the three 3xTF32 products (tc.cuh) costs 5.7e-5 or more on every launch that
uses that contraction, and a wrong halo row at a band edge costs 1e-1."""
import json
import re
import time

import pytest
import torch

import yfv2  # noqa: F401
import synth
import net_dispatch as nd
from oracle import net as onet

# one bound for every launch, and a looser one for the six head tensors after all 21 launches against a full fp64 forward
BOUND = 1.2e-5
E2E_BOUND = 1.5e-5

# name -> (N, H, W, anchors, classes, images checked against fp64)
CASES = {
    "1x32x32": (1, 32, 32, 3, 80, None),               # every map at its minimum, partial 16-pixel tiles, every stage chained
    "2x64x96": (2, 64, 96, 3, 80, None),               # the shape of tests/golden/net_small.npz
    "1x32x640": (1, 32, 640, 3, 80, None),             # one-pixel-tall maps at stride 32; chain96
    "1x640x32": (1, 640, 32, 3, 80, None),             # one-pixel-wide maps at stride 32 (Wt = 3)
    "16x352": (16, 352, 352, 3, 80, (0, 5, 15)),       # first multi-row stage-2 bands
    "64x352": (64, 352, 352, 3, 80, (0, 31, 63)),      # partial last bands in stages 2-3
    "8x512x256": (8, 512, 256, 3, 80, (0, 7)),         # stage4.0 whole-image at Ho*Wo = 128
    "8x544x256": (8, 544, 256, 3, 80, (0, 7)),         # stage4.0 banded at 136
    "1x640": (1, 640, 640, 3, 80, None),               # R = 1 everywhere, stage4.1-3 banded and unchained
    "128x640": (128, 640, 640, 3, 80, (0, 63, 64, 127)),   # bench.py --side 640 geometry
    "24x832x160": (24, 832, 160, 3, 80, (0, 23)),      # stage4.0 banded, R > 1
    "24x864x160": (24, 864, 160, 3, 80, (0, 23)),      # stage4.0 banded, R > 1, partial last band
    "24x960x320": (24, 960, 320, 3, 80, (0, 23)),      # stage4.1-3 banded blk_kernel<96, 1>, R > 1
    "24x992x320": (24, 992, 320, 3, 80, (0, 23)),      # the same with a partial last band
    "2x96x128c150": (2, 96, 128, 3, 150, None),        # head2_kernel
    "2x128x128a2c20": (2, 128, 128, 2, 20, None),      # other anchor and class counts
}
SEED = {name: 1000 + 10 * i for i, name in enumerate(CASES)}


def case_cells(sms):
    out = set()
    for n, h, w, a, c, _ in CASES.values():
        out |= nd.cells(n, h, w, a, c, sms)
    return out


def test_cases_cover_every_reachable_cell():
    """With 132 SMs (H100 SXM), the cases reach every cell any plan of the dispatch model's search space reaches."""
    assert set(nd.reachable(132)) == nd.ALL_CELLS
    missing = nd.ALL_CELLS - case_cells(132)
    assert not missing, {cl: nd.find_case(cl, 132) for cl in missing}


@pytest.mark.gpu
def test_cases_cover_every_reachable_cell_on_this_device():
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    missing = set(nd.reachable(sms)) - case_cells(sms)
    assert not missing, {cl: nd.find_case(cl, sms) for cl in missing}


def sm_count():
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


def setup(name):
    import model.detector as det
    n, h, w, a, c, imgs = CASES[name]
    sd = synth.make_state_dict(SEED[name], classes=c, anchor_num=a)
    m = det.Detector(c, a, True)
    m.load_state_dict(sd, strict=True)
    m = m.cuda().eval()
    x = synth.make_images(SEED[name] + 1, n, h, w).cuda()
    imgs = list(range(n)) if imgs is None else list(imgs)
    return m, sd, x, imgs


def io_taps(L):
    """debug_gather ids a launch reads and writes; 'preds' for the head tensors of a level."""
    name = L.names[0]
    if name == "stem":
        return [], [0]
    if L.blocks:
        return [L.blocks[0]], [L.blocks[-1] + 1]          # id b + 1 is the output of block b, id 0 the stem's
    return {"fpn.S3": ([16], [18]), "fpn.S2": ([12, 16], [17]), "heads2.a": ([17], [19, 20]), "heads2.b": ([19, 20], "preds"),
            "heads3.a": ([18], [21, 22]), "heads3.b": ([21, 22], "preds")}[name]


def reference(L, sd, ins):
    """The fp64 oracle of exactly this launch."""
    name = L.names[0]
    if name == "stem":
        return [onet.stem(sd, ins[0])]
    if L.blocks:
        y = ins[0]
        for b in L.blocks:
            bname, _, stride, _ = nd.BLOCKS[b]
            y = onet.shuffle_block(sd, y, "backbone.%s." % bname, stride)
        return [y]
    if name == "fpn.S3":
        return [onet.reduce_s3(sd, ins[0])]
    if name == "fpn.S2":
        return [onet.reduce_s2(sd, ins[0], ins[1])]
    lv = int(name[5])
    cls, reg = "fpn.cls_head_%d." % lv, "fpn.reg_head_%d." % lv
    if name.endswith(".a"):
        return [onet.dwconv_half(sd, ins[0], cls, 0), onet.dwconv_half(sd, ins[0], reg, 0)]
    return list(onet.output_layers(sd, onet.dwconv_half(sd, ins[0], cls, 1), onet.dwconv_half(sd, ins[1], reg, 1)))


def nerr(got, ref):
    """max over the images of max|got - ref| / max(max|ref|, 1e-3)"""
    d = (got - ref).abs().flatten(1).max(1).values
    s = ref.abs().flatten(1).max(1).values.clamp_min(1e-3)
    return (d / s).max().item()


def gather(plan, which, idx):
    g = plan.debug_gather(which)
    out = g[idx].double().cpu()
    del g
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_every_launch_against_fp64(name):
    m, sd, x, imgs = setup(name)
    n, h, w, a, c, _ = CASES[name]
    sd64 = {k: v.double() if v.is_floating_point() else v for k, v in sd.items()}
    idx = torch.tensor(imgs, device="cuda")
    preds = m(x)
    full = [p[idx].double().cpu() for p in preds]
    plan = next(iter(m._plans.values()))
    model = nd.launches(n, h, w, a, c, sm_count())
    assert plan.stage_names == nd.STAGE_NAMES and plan.stage_groups == nd.stage_groups(h, w)
    assert plan.forward_launches == len(model)
    x64 = x[idx].double().cpu()
    rows = []
    for L in model:
        tin, tout = io_taps(L)
        ins = [gather(plan, t, idx) for t in tin] if tin else [x64]
        plan.forward_range(x, preds, L.first, L.last)
        if tout == "preds":
            lv = int(L.names[0][5]) - 2
            got = [p[idx].double().cpu() for p in preds[3 * lv:3 * lv + 3]]
        else:
            got = [gather(plan, t, idx) for t in tout]
        ref = reference(L, sd64, ins)
        assert [g.shape for g in got] == [r.shape for r in ref], L.names
        rows.append((L, max(nerr(g, r) for g, r in zip(got, ref))))
    # the stem again, on uint8 pixels: the reference divides by 255 in fp64
    xu8 = (x * 255).to(torch.uint8)
    plan.forward_range(xu8, preds, 0, 1)
    L = nd.launches(n, h, w, a, c, sm_count(), u8=True)[0]
    rows.append((L, nerr(gather(plan, 0, idx), onet.stem(sd64, xu8[idx].double().cpu() / 255))))
    with torch.no_grad():
        ref = onet.forward(sd64, x64)
    e2e = max(nerr(g, r) for g, r in zip(full, ref))
    print("\n%s (N=%d, %dx%d, A=%d, C=%d), images %s" % (name, n, h, w, a, c, imgs))
    for L, e in rows:
        geo = "R=%d bands=%d%s" % (L.R, L.bands, " partial" if L.partial else "") if L.bands else ""
        print("  %-22s %-24s %-16s %-24s %.3e" % ("%s..%s" % (L.names[0], L.names[-1]) if len(L.names) > 1 else L.names[0],
                                                   L.kernel, L.variant, geo, e))
    print("  %-22s %-24s %-16s %-24s %.3e" % ("end to end", "", "", "", e2e))
    bad = [(L.names[0], L.kernel, L.variant, e) for L, e in rows if not e <= BOUND]
    assert not bad, bad
    assert e2e <= E2E_BOUND, e2e


KERNEL_RE = re.compile(r"\b(stem_kernel|blk_kernel|blk_s2_image_kernel|blk_chain_kernel|fpn_kernel|head_kernel|head2_kernel)(<[^>]*>)?")
# The activity tracer keeps only device records whose timestamps, converted to the host clock, fall inside the session's
# window; a forward of microsecond kernels recorded right at a window edge can lose records to that conversion.  The recorded
# forward therefore sits in the middle of its session, with this much idle host time on either side.
TRACE_MARGIN_S = 0.05


@pytest.fixture(scope="module")
def tracer_ready():
    """One throw-away CUDA activity session before any recorded one: the first session of a process initialises the tracer."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]):
        torch.ones(1, device="cuda").add_(1)
        torch.cuda.synchronize()


def traced_launches(fn, path):
    """Runs fn() in one CUDA activity session and returns this project's kernel launches in launch order, as
    (kernel, grid, correlation id, start ts) tuples.  Every kernel launch call the session recorded must have its kernel."""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        time.sleep(TRACE_MARGIN_S)
        fn()
        torch.cuda.synchronize()
        time.sleep(TRACE_MARGIN_S)
    prof.export_chrome_trace(str(path))
    events = json.load(open(path))["traceEvents"]
    calls = {e["args"]["correlation"]: e for e in events
             if e.get("cat") == "cuda_runtime" and e.get("name", "").startswith("cudaLaunchKernel")}
    kernels = {e["args"]["correlation"]: e for e in events if e.get("cat") == "kernel"}
    lost = sorted(set(calls) - set(kernels))
    assert not lost, "the trace recorded launch calls without their kernels: correlation ids %s of %s" % (lost, sorted(calls))
    out = []
    for corr in sorted(kernels):
        e = kernels[corr]
        k = KERNEL_RE.search(e["name"])
        if k:
            out.append((k.group(0).replace(" ", ""), tuple(e["args"]["grid"]), corr, e["ts"]))
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_launches_match_the_dispatch_model(name, tmp_path, tracer_ready):
    """Kernel names and, where the host code fixes them, grids of one forward, from a CUDA activity trace."""
    m, _, x, _ = setup(name)
    n, h, w, a, c, _ = CASES[name]
    preds = m(x)
    plan = next(iter(m._plans.values()))
    got = traced_launches(lambda: plan.forward(x, preds), tmp_path / "forward.json")
    sms = sm_count()
    model = nd.launches(n, h, w, a, c, sms)
    table = "\n".join("  corr %d ts %.1f %s grid %s" % (corr, ts, k, grid) for k, grid, corr, ts in got)
    assert [k for k, _, _, _ in got] == [L.kernel for L in model], "model %s, trace:\n%s" % ([L.kernel for L in model], table)
    for L, (_, grid, _, _) in zip(model, got):
        if L.grid is not None:
            assert grid == L.grid, (L.names, grid, L.grid, table)
        else:                                 # persistent grid sized by occupancy: at least one CTA per SM, at most one per item
            assert min(L.items, sms) <= grid[0] <= L.items and grid[1:] == (1, 1), (L.names, grid, L.items, table)


@pytest.mark.gpu
def test_batch_128_at_640_equals_images_alone():
    """The 640 counterpart of the 352 batch-invariance test: in the 128 x 640^2 forward (R = 2 / 11 partial / 2 / 8 bands in
    stages 2-3), each checked image equals, bit for bit, the same image run alone, where every band has one row."""
    m, _, x, imgs = setup("128x640")
    big = [p.clone() for p in m(x)]
    assert {L.R for L in nd.launches(1, 640, 640, sms=sm_count()) if L.bands} == {1}
    for i in imgs:
        one = m(x[i:i + 1])
        for p, q in zip(big, one):
            assert torch.equal(p[i], q[0]), i
