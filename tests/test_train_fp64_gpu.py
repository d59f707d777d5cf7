"""Every op of the native trainer's program (csrc/trainer.cu), forward and backward, against an fp64 restatement of the same op,
fed what the GPU consumed.

One training step per case runs on the native trainer (train-mode forward, utils.loss.compute_loss, backward); every activation and
gradient stays in the trainer's workspace, which yfv2_trainer_debug_ops / _tensors map.  Each op is then recomputed in float64 from
the fp32 tensors it read (its input, the output gradient the GPU held, for BatchNorm + ReLU the GPU's own y as the mask and the
saved mean / invstd), so error does not compound and one elementwise bound holds for every op:

    |got - ref| <= TAU * mag

where mag is the same op in fp64 over absolute values (|W|.|X|, |dY|^T.|X|, ...), and for BatchNorm the sum of the absolute values
of the terms the kernel adds: forward (|x - mu| + |mu|) invstd |gamma| + |beta| (the |mu| term covers the fp32 rounding of mu),
backward |gamma| invstd (|d| + mean|d| + |xhat| mean|d xhat|).  The gradient of a tensor with several consumers is checked against
the sum of every consumer's fp64 dgrad, each parameter's slot of the flat buffer against the sum of its uses (both levels of the
shared output convolutions), the saved statistics and the running-stat update (momentum 0.1, unbiased variance) against fp64.
Channel copies and up-sampling are checked bit for bit, max-pool values and indices against torch CUDA's max_pool2d.  A second
backward with accumulate=1 must add the same gradients again (fp32 atomics: within the bound, not bit for bit).

Measured on an H100 80GB HBM3 (132 SMs, 700 W power limit), the worst |got - ref| / mag over every op of every case (and of
tests/test_train_ops_space_gpu.py) is 6.4e-7; TAU sits 3.1x above it.  Deliberate faults fail it by far: one 32-pixel slab skipped in
wgrad1x1_kernel 0.47, one slice dropped in wgrad_reduce_kernel 1.0, the stride-2 row test of dw_dgrad_kernel off by one 1.5e8, even
and odd swapped in the K_CATE backward (bit-exact check), the ReLU mask dropped in bn_bwd_apply_kernel 6.7e32, the biased variance
in the running-var update 0.36.  tests/train_dispatch.py maps which kernel variants each case reaches."""
import collections

import pytest
import torch
import torch.nn.functional as F

import yfv2  # noqa: F401
import synth
import train_dispatch as td

TAU = 2e-6                       # one bound for every op (measured worst 6.4e-7, see above)

# name -> (N, H, W, anchors, classes)
CASES = {
    "2x32x32": (2, 32, 32, 3, 80),               # 1x1 maps at stride 32, 5x5 heads over 1x1 and 2x2 maps
    "1x32x64": (1, 32, 64, 3, 80),               # N = 1, two values per stride-32 BatchNorm
    "3x64x96": (3, 64, 96, 3, 80),               # odd maps (2x3 at stride 32), scalar HW%4 paths
    "2x640x352": (2, 640, 352, 3, 80),           # non-square, odd 11-column maps, BN apply y-grid > 1
    "64x352": (64, 352, 352, 3, 80),             # bench.py --mode train: multi-chunk wgrad, partial reduce, 64 BN slices
    "203x32x32": (203, 32, 32, 3, 80),           # past the partial-scratch limit: fpn.conv1x1_2 wgrad by memset + atomics
    "2x96x128c150": (2, 96, 128, 3, 150),        # wide class convolution
    "2x64x64c300": (2, 64, 64, 3, 300),          # weight + bias of the class conv above every other parameter (pscratch)
    "2x128x128a2c20": (2, 128, 128, 2, 20),      # other anchor and class counts
}
SEED = {name: 2000 + 10 * i for i, name in enumerate(CASES)}
CPU_CHECK_CASE = "2x32x32"       # its fp64 references are recomputed on the CPU and must agree to 1e-12
EPS = 1e-5
KINDS_COPY = ("odd", "cate", "cat2")


def case_cells(sms):
    out = set()
    for n, h, w, a, c in CASES.values():
        out |= td.trainer_cells(n, h, w, a, c, sms)
    return out


@pytest.mark.gpu
def test_cases_cover_every_reachable_trainer_cell_on_this_device():
    import test_train_ops_space_gpu as sp
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    have = case_cells(sms) | sp.case_cells(sms)
    missing = (set(td.reachable(sms)) | (td.ALL_CELLS - td.TRAINER_ONLY)) - have
    assert not missing, {cl: td.find_case(cl, sms) for cl in missing}
    only = set(td.reachable(sms)) & td.TRAINER_ONLY
    assert only <= case_cells(sms), only - case_cells(sms)


# ---- fp64 references of one op: pure functions of float64 tensors (device-agnostic) ---------------------------------------------
def ref_op(kind, o, t):
    """t: float64 inputs (x, b, y, dy, w, bias, gamma, beta, mean, invstd, idx) -> {name: (ref, mag)}"""
    out = {}
    x, dy = t["x"], t["dy"]
    if kind == "stem":
        w = t["w"]
        out["y"] = (F.conv2d(x, w, None, 2, 1), F.conv2d(x.abs(), w.abs(), None, 2, 1))
        out["dw"] = (torch.nn.grad.conv2d_weight(x, w.shape, dy, 2, 1), torch.nn.grad.conv2d_weight(x.abs(), w.shape, dy.abs(), 2, 1))
    elif kind == "pw":
        N, K = x.shape[:2]
        w = t["w"].reshape(t["w"].shape[0], K)
        X, D = x.reshape(N, K, -1), dy.reshape(N, w.shape[0], -1)
        y, ym = torch.einsum("mk,nkp->nmp", w, X), torch.einsum("mk,nkp->nmp", w.abs(), X.abs())
        if t.get("bias") is not None:
            y, ym = y + t["bias"].view(1, -1, 1), ym + t["bias"].abs().view(1, -1, 1)
        out["y"] = (y.reshape(N, -1, *x.shape[2:]), ym.reshape(N, -1, *x.shape[2:]))
        out["dx"] = (torch.einsum("mk,nmp->nkp", w, D).reshape(x.shape), torch.einsum("mk,nmp->nkp", w.abs(), D.abs()).reshape(x.shape))
        out["dw"] = (torch.einsum("nmp,nkp->mk", D, X).reshape(t["w"].shape), torch.einsum("nmp,nkp->mk", D.abs(), X.abs()).reshape(t["w"].shape))
        if t.get("bias") is not None:
            out["dbias"] = (D.sum((0, 2)), D.abs().sum((0, 2)))
    elif kind == "dw":
        w, s = t["w"], o["stride"]
        C, p = x.shape[1], o["ks"] // 2
        out["y"] = (F.conv2d(x, w, None, s, p, 1, C), F.conv2d(x.abs(), w.abs(), None, s, p, 1, C))
        out["dx"] = (torch.nn.grad.conv2d_input(x.shape, w, dy, s, p, 1, C), torch.nn.grad.conv2d_input(x.shape, w.abs(), dy.abs(), s, p, 1, C))
        out["dw"] = (torch.nn.grad.conv2d_weight(x, w.shape, dy, s, p, 1, C), torch.nn.grad.conv2d_weight(x.abs(), w.shape, dy.abs(), s, p, 1, C))
    elif kind == "bn":
        g, b = t["gamma"].view(1, -1, 1, 1), t["beta"].view(1, -1, 1, 1)
        cnt = x.numel() // x.shape[1]
        mu = x.mean((0, 2, 3))
        var = (x - mu.view(1, -1, 1, 1)).square().mean((0, 2, 3))
        ex2 = x.square().mean((0, 2, 3))
        inv = 1.0 / torch.sqrt(var + EPS)
        cancel = 1.0 + 2.0 ** -24 * ex2 / (var + EPS)                # the E[x^2] - mu^2 variance of the kernel, at fp32 precision
        out["mean"] = (mu, x.abs().mean((0, 2, 3)))
        out["invstd"] = (inv, inv * cancel)
        out["var_unbiased"] = (var * cnt / (cnt - 1), var * cnt / (cnt - 1) * cancel)
        m4, i4 = mu.view(1, -1, 1, 1), inv.view(1, -1, 1, 1)
        y = (x - m4) * i4 * g + b
        ym = ((x - m4).abs() + m4.abs()) * i4 * g.abs() + b.abs()
        if o["relu"]:
            y = y.clamp_min(0)
        out["y"] = (y, ym)
        ms, iss = t["mean"].view(1, -1, 1, 1), t["invstd"].view(1, -1, 1, 1)
        d = torch.where(t["y"] <= 0, torch.zeros_like(dy), dy) if o["relu"] else dy      # threshold_backward on the GPU's y
        xh = (x - ms) * iss
        sd, sdx = d.mean((0, 2, 3), keepdim=True), (d * xh).mean((0, 2, 3), keepdim=True)
        out["dx"] = (g * iss * (d - sd - xh * sdx),
                     g.abs() * iss * (d.abs() + d.abs().mean((0, 2, 3), keepdim=True) + xh.abs() * (d * xh).abs().mean((0, 2, 3), keepdim=True)))
        out["dgamma"] = ((d * xh).sum((0, 2, 3)), (d * xh).abs().sum((0, 2, 3)))
        out["dbeta"] = (d.sum((0, 2, 3)), d.abs().sum((0, 2, 3)))
    elif kind == "pool":
        N, C, H, W = x.shape
        idx = t["idx"].reshape(N, C, -1)
        z = torch.zeros(N, C, H * W, dtype=dy.dtype, device=dy.device)
        out["dx"] = (z.scatter_add(2, idx, dy.reshape(N, C, -1)).view(x.shape), z.scatter_add(2, idx, dy.abs().reshape(N, C, -1)).view(x.shape))
    elif kind == "up":
        N, C, H, W = x.shape
        d = dy.view(N, C, H, 2, W, 2)
        out["dx"] = (d.sum((3, 5)), d.abs().sum((3, 5)))
    return out


def nerr(got, ref, mag):
    """max |got - ref| / mag (mag = 0 only where ref is exactly 0: any nonzero got there is an error); NaN counts as infinite"""
    e = (got.double() - ref).abs() / mag.clamp_min(1e-30)
    e = torch.where(torch.isnan(e), torch.full_like(e, float("inf")), e)
    return float(e.max()) if e.numel() else 0.0


# ---- one training step, every op checked --------------------------------------------------------------------------------------
def run_step(name, m=None):
    """one training step of case `name`; m: the model of an earlier run_step of the case, to step its trainer again"""
    import model.detector as det
    import utils.loss as ul
    n, h, w, a, c = CASES[name]
    if m is None:
        sd = synth.make_state_dict(SEED[name], classes=c, anchor_num=a)
        m = det.Detector(c, a, True)
        m.load_state_dict(sd, strict=True)
        m = m.cuda().train()
    x = synth.make_images(SEED[name] + 1, n, h, w).cuda()
    targets = synth.make_targets(SEED[name] + 2, n, classes=c).cuda()
    cfg = synth.coco_cfg(w, h, c)
    cfg["anchor_num"] = a
    cfg["anchors"] = (synth.COCO_ANCHORS if a == 3 else [float(8 + 7 * i) for i in range(4 * a)])
    bn_before = [t.clone() for t in m._train_buffers()[0]]
    preds = m(x)
    ul.compute_loss(preds, targets, cfg, x.device)[3].backward()
    torch.cuda.synchronize()
    return m, m._trainer_for(x), bn_before


class Checker:
    def __init__(self, case):
        self.case = case
        self.rows = collections.defaultdict(float)          # site -> worst normalised error
        self.exact_fail = []

    def check(self, site, got, ref, mag):
        e = nerr(got, ref, mag)
        self.rows[site] = max(self.rows[site], e)
        return e

    def exact(self, site, ok):
        self.rows[site] = max(self.rows[site], 0.0 if ok else float("inf"))
        if not ok:
            self.exact_fail.append(site)


def site_name(o, tens):
    c, h, w = tens[o["a"]]["C"], tens[o["a"]]["H"], tens[o["a"]]["W"]
    extra = {"pw": " M=%d" % o["M"], "dw": " %dx%d s%d" % (o["ks"], o["ks"], o["stride"]), "bn": " relu" if o["relu"] else ""}.get(o["kind"], "")
    return "%s %dx%dx%d%s" % (o["kind"], c, h, w, extra)


def check_case(name, cpu_check=False, step=None):
    """step: what run_step(name) returned, to check that step instead of running one"""
    n, h, w, a, c = CASES[name]
    m, tr, bn_before = step or run_step(name)
    ops, tens, layout = tr.program()
    assert [o["kind"] for o in ops] == [o["kind"] for o in td.program(n, h, w, a, c)[0]]
    params = [p.detach() for p in m.parameters()]
    bn_after = m._train_buffers()[0]
    wsf = tr.workspace.view(torch.float32)
    wsi = tr.workspace.view(torch.int32)
    cons = td.consumers(ops, len(tens))

    def act(i):
        T = tens[i]
        if T["ext"] == -2:
            return tr.x_static
        if T["ext"] >= 0:
            return tr.preds_static[T["ext"]]
        return wsf[T["off"]:T["off"] + n * T["C"] * T["H"] * T["W"]].view(n, T["C"], T["H"], T["W"])

    def grad(i):
        T = tens[i]
        if T["ext"] >= 0:
            return tr.dpreds_static[T["ext"]]
        return wsf[T["goff"]:T["goff"] + n * T["C"] * T["H"] * T["W"]].view(n, T["C"], T["H"], T["W"])

    flat = tr.flat_static.clone()
    ck = Checker(name)
    gacc = {}                                    # tensor id -> [ref, mag] of its gradient, summed over its consumers
    pacc = {}                                    # parameter index -> [ref, mag]
    cpu_worst, cpu_checked = 0.0, set()

    def add(dct, key, ref, mag):
        if key in dct:
            dct[key][0] += ref; dct[key][1] += mag
        else:
            dct[key] = [ref.clone(), mag.clone()]

    for i in range(len(ops) - 1, -1, -1):       # backward order: when op i is reached, its output's gradient is complete
        o = ops[i]
        k, site = o["kind"], site_name(o, tens)
        Y = tens[o["y"]]
        if Y["ext"] == -1:
            r, mg = gacc.pop(o["y"])
            if all(ops[j]["kind"] in KINDS_COPY for j in cons[o["y"]]) and \
                    (len(cons[o["y"]]) == 1 or {ops[j]["kind"] for j in cons[o["y"]]} == {"odd", "cate"}):
                ck.exact(site + " / dx (copies)", torch.equal(grad(o["y"]).double(), r))
            else:
                ck.check(site + " / dx", grad(o["y"]), r, mg)
        xa, dy, ya = act(o["a"]), grad(o["y"]), act(o["y"])
        if k in KINDS_COPY or k == "up":
            xb = act(o["b"]) if o["b"] >= 0 else None
            if k == "odd":
                ck.exact(site + " / fwd", torch.equal(ya, xa[:, 1::2]))
                z = torch.zeros(xa.shape, dtype=torch.float64, device="cuda"); z[:, 1::2] = dy.double()
                add(gacc, o["a"], z, z.abs())
            elif k == "cate":
                ck.exact(site + " / fwd", torch.equal(ya, torch.cat((xa[:, 0::2], xb), 1)))
                z = torch.zeros(xa.shape, dtype=torch.float64, device="cuda"); z[:, 0::2] = dy[:, :xa.shape[1] // 2].double()
                add(gacc, o["a"], z, z.abs())
                zb = dy[:, xa.shape[1] // 2:].double()
                add(gacc, o["b"], zb, zb.abs())
            elif k == "cat2":
                ck.exact(site + " / fwd", torch.equal(ya, torch.cat((xa, xb), 1)))
                za, zb = dy[:, :xa.shape[1]].double(), dy[:, xa.shape[1]:].double()
                add(gacc, o["a"], za, za.abs())
                add(gacc, o["b"], zb, zb.abs())
            else:
                ck.exact(site + " / fwd", torch.equal(ya, xa.repeat_interleave(2, 2).repeat_interleave(2, 3)))
                r = ref_op("up", o, {"x": xa.double(), "dy": dy.double()})["dx"]
                add(gacc, o["a"], *r)
            continue
        t = {"x": xa.double(), "dy": dy.double(), "y": ya.double()}
        if k == "pool":
            yt, it = F.max_pool2d(xa, 3, 2, 1, return_indices=True)
            gidx = wsi[o["aux"]:o["aux"] + ya.numel()].view(ya.shape)
            ck.exact(site + " / fwd values", torch.equal(ya, yt))
            ck.exact(site + " / fwd indices", torch.equal(gidx.long(), it))
            t["idx"] = gidx.long()
        if o["pw"] >= 0:
            t["w"] = params[o["pw"]].double()
        if o["pbias"] >= 0:
            t["bias"] = params[o["pbias"]].double()
        if k == "bn":
            C = xa.shape[1]
            t["gamma"], t["beta"] = params[o["pg"]].double(), params[o["pb"]].double()
            t["mean"] = wsf[o["aux"] + 4 * C:o["aux"] + 5 * C].double()
            t["invstd"] = wsf[o["aux"] + 5 * C:o["aux"] + 6 * C].double()
        R = ref_op(k, o, t)
        if cpu_check and (k, o["ks"], o["stride"], o["relu"]) not in cpu_checked:      # the first op of each variant
            cpu_checked.add((k, o["ks"], o["stride"], o["relu"]))
            threads = torch.get_num_threads()
            torch.set_num_threads(1)                 # (tiny grouped fp64 convolutions crawl on a many-core pool)
            try:
                Rc = ref_op(k, o, {kk: v.cpu() if v is not None else None for kk, v in t.items()})
            finally:
                torch.set_num_threads(threads)
            for kk, (r, mg) in R.items():
                cpu_worst = max(cpu_worst, nerr(Rc[kk][0], r.cpu(), mg.cpu().abs() + r.cpu().abs()))
        if "y" in R:
            ck.check(site + " / fwd", ya, *R["y"])
        if k == "bn":
            ck.check(site + " / saved mean", t["mean"], *R["mean"])
            ck.check(site + " / saved invstd", t["invstd"], *R["invstd"])
            rm0, rv0 = bn_before[2 * o["bn"]].double(), bn_before[2 * o["bn"] + 1].double()
            mu, mmag = R["mean"]
            vu, vmag = R["var_unbiased"]
            ck.check(site + " / running_mean", bn_after[2 * o["bn"]], 0.9 * rm0 + 0.1 * mu, 0.9 * rm0.abs() + 0.1 * mmag)
            ck.check(site + " / running_var", bn_after[2 * o["bn"] + 1], 0.9 * rv0 + 0.1 * vu, 0.9 * rv0.abs() + 0.1 * vmag)
            add(pacc, o["pg"], *R["dgamma"])
            add(pacc, o["pb"], *R["dbeta"])
        if "dw" in R:
            add(pacc, o["pw"], *R["dw"])
        if "dbias" in R:
            add(pacc, o["pbias"], *R["dbias"])
        if "dx" in R and tens[o["a"]]["ext"] == -1:
            add(gacc, o["a"], *R["dx"])
        del t, R
    assert not gacc, sorted(gacc)
    assert sorted(pacc) == list(range(len(params)))
    offs = tr.param_offsets
    for pi, (r, mg) in pacc.items():
        off, num = offs[pi]
        ck.check("param %03d %s" % (pi, tuple(params[pi].shape)), flat[off:off + num].view(params[pi].shape), r, mg)
    # gradient accumulation: a second backward of the same batch adds the same gradients to the flat buffer
    acc = flat.clone()
    tr.backward(params, list(tr.dpreds_static), acc, accumulate=True)
    torch.cuda.synchronize()
    worst_acc = 0.0
    for pi, (r, mg) in pacc.items():
        off, num = offs[pi]
        worst_acc = max(worst_acc, nerr((acc[off:off + num] - flat[off:off + num]).view(params[pi].shape), r, mg + flat[off:off + num].view(params[pi].shape).abs().double()))
    ck.rows["accumulate=1: second backward"] = worst_acc
    return ck, cpu_worst, layout


def report(name, ck):
    n, h, w, a, c = CASES[name]
    print("\n%s (N=%d, %dx%d, A=%d, C=%d)" % (name, n, h, w, a, c))
    by_site = ck.rows
    worst_param = max((e for s, e in by_site.items() if s.startswith("param")), default=0.0)
    for s in sorted(k for k in by_site if not k.startswith("param")):
        print("  %-60s %.3e" % (s, by_site[s]))
    print("  %-60s %.3e" % ("parameter slots of the flat buffer (worst)", worst_param))
    worst = max(by_site.values())
    print("  %-60s %.3e   (tau %.1e)" % ("worst in case", worst, TAU))
    return worst


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_every_trainer_op_against_fp64(name):
    ck, cpu_worst, layout = check_case(name, cpu_check=(name == CPU_CHECK_CASE))
    report(name, ck)
    assert not ck.exact_fail, ck.exact_fail
    bad = sorted((s, e) for s, e in ck.rows.items() if not e <= TAU)
    assert not bad, bad[:20]
    if name == CPU_CHECK_CASE:
        print("  fp64 references on the GPU against the CPU: %.3e" % cpu_worst)
        assert cpu_worst <= 1e-12
