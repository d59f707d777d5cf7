"""The yfv2_op_* training entries (csrc/k_train.cu) over their whole dispatch space, one op per call, against the fp64 references
and the elementwise bound of tests/test_train_fp64_gpu.py.  This covers the cells the native trainer never reaches
(tests/train_dispatch.py): base pointers only 4-byte aligned, HW%4 != 0, K = 24 with M = 48 / 72, the generic stem, 5x5 at
stride 2, H or W = 1, maps smaller than the stencil, N > 16, HW > 1024, 64 BatchNorm slices, a large mean over a small spread;
and the special values where the kernels must do what torch does: NaN and +-inf through BatchNorm + ReLU and max-pool, exact ties
and all-equal windows, and the refusal of a BatchNorm over one value per channel."""
import pytest
import torch
import torch.nn.functional as F

import yfv2  # noqa: F401
import train_dispatch as td
from test_train_fp64_gpu import TAU, nerr, ref_op

# conv1x1: (N, K, M, H, W, bias, storage offset of every tensor)
PW = [(2, 24, 24, 8, 8, False, 0),       # wgrad rows, one chunk, BM = 32
      (3, 24, 48, 5, 7, False, 0),       # rows with blockIdx.y > 0, HW % 4 != 0
      (2, 24, 72, 40, 40, True, 0),      # rows, three row groups, several pixel chunks
      (2, 16, 16, 8, 8, False, 0),       # tiled32, one chunk
      (2, 16, 16, 9, 9, False, 0),       # tiled32, several chunks, HW % 4 != 0
      (2, 72, 80, 4, 4, True, 0),        # tiled64, one chunk, bias
      (4, 96, 96, 30, 30, False, 0),     # tiled64, several chunks
      (2, 48, 72, 8, 8, False, 1),       # B and C of both GEMMs only 4-byte aligned
      (1, 3, 5, 1, 1, True, 1)]          # one pixel
# depthwise: (N, C, H, W, ks, stride)
DW = [(2, 8, 7, 9, 3, 1), (2, 8, 7, 9, 3, 2), (2, 8, 9, 6, 5, 2), (3, 8, 2, 1, 5, 1), (2, 4, 1, 5, 3, 2), (20, 4, 6, 5, 3, 1),
      (17, 3, 4, 4, 5, 2), (2, 5, 3, 3, 5, 1)]
# BatchNorm: (N, C, H, W, relu, mean, spread, storage offset)
BN = [(3, 5, 7, 9, True, 0.0, 1.0, 0),        # scalar access
      (2, 4, 40, 40, False, 0.5, 2.0, 0),     # HW > 1024: apply y-grid 2, float4
      (200, 3, 40, 40, True, 0.0, 1.0, 0),    # 64 slices (the cap)
      (4, 6, 16, 16, True, 50.0, 0.5, 0),     # large mean over a small spread
      (1, 3, 1, 2, True, 0.0, 1.0, 0),        # two values per channel
      (2, 4, 8, 8, True, 0.0, 1.0, 1)]        # 4-byte aligned: scalar paths
# stem: (N, M, H, W)
STEM = [(2, 24, 16, 18), (2, 10, 8, 12), (1, 8, 6, 2)]
# max-pool / up-sampling: (N, C, H, W)
POOL = [(2, 3, 7, 9), (1, 2, 6, 8), (2, 2, 1, 1)]
UP = [(2, 3, 5, 7), (1, 2, 1, 1)]


def case_cells(sms):
    """The cells the op calls of this suite reach, from the library's records of those calls (yfv2_op_debug_launches) at the
    addresses buf() / empty() give: a 256-byte-aligned allocation, `off` floats into it."""
    at = lambda off: (1 << 20) + 4 * off
    a0 = at(0)
    out = set()
    for n, k, m, h, w, bias, off in PW:
        p = at(off)
        out |= td.op_cells("conv1x1_fwd", [p, p, p if bias else None, p], [n, k, m, h * w], sms)
        out |= td.op_cells("conv1x1_bwd", [p, p, p, p, p, p if bias else None], [n, k, m, h * w], sms)
    for n, c, h, w, ks, s in DW:
        out |= td.op_cells("dwconv_fwd", [a0] * 3, [n, c, h, w, ks, s], sms)
        out |= td.op_cells("dwconv_bwd", [a0] * 5, [n, c, h, w, ks, s], sms)
    for n, c, h, w, relu, _, _, off in BN:
        p = at(off)
        out |= td.op_cells("bn_train_fwd", [p, a0, a0, a0, a0, p, a0, a0, a0], [n, c, h * w, int(relu)], sms)
        out |= td.op_cells("bn_train_bwd", [p, p, p, a0, a0, a0, p, a0, a0, a0], [n, c, h * w, int(relu)], sms)
    for n, m, h, w in STEM:
        out |= td.op_cells("stem_fwd", [a0] * 3, [n, m, h, w], sms)
        out |= td.op_cells("stem_wgrad", [a0] * 3, [n, m, h, w], sms)
    for n, c, h, w in POOL:
        out |= td.op_cells("maxpool_fwd", [a0] * 3, [n * c, h, w], sms)
        out |= td.op_cells("maxpool_bwd", [a0] * 3, [n * c, h, w], sms)
    for n, c, h, w in UP:
        out |= td.op_cells("upsample2_fwd", [a0] * 2, [n * c, h, w], sms)
        out |= td.op_cells("upsample2_bwd", [a0] * 2, [n * c, h, w], sms)
    return out


def op(name, args):
    import yfv2_engine as eng
    eng.op(name, args, torch.device("cuda"))


def buf(shape, off, gen, scale=1.0, shift=0.0):
    """a float32 tensor of `shape` starting `off` floats into its storage (off = 1: only 4-byte aligned)"""
    n = 1
    for s in shape:
        n *= s
    base = torch.randn(n + off, device="cuda", generator=gen) * scale + shift
    return base[off:].view(shape)


def empty(shape, off):
    n = 1
    for s in shape:
        n *= s
    return torch.full((n + off,), float("nan"), device="cuda")[off:].view(shape)


def check_all(name, checks):
    bad = [(k, e) for k, e in checks if not e <= TAU]
    print("  %-44s %s" % (name, "  ".join("%s %.2e" % kv for kv in checks)))
    assert not bad, (name, bad)


@pytest.mark.gpu
@pytest.mark.parametrize("case", PW, ids=lambda c: "N%d_K%d_M%d_%dx%d%s%s" % (c[0], c[1], c[2], c[3], c[4], "_bias" if c[5] else "", "_off%d" % c[6] if c[6] else ""))
def test_conv1x1(case):
    n, k, m, h, w, bias, off = case
    g = torch.Generator(device="cuda").manual_seed(hash(case) % 2 ** 31)
    x = buf((n, k, h, w), off, g)
    wt = buf((m, k, 1, 1), off, g, k ** -0.5)
    b = buf((m,), off, g) if bias else None
    dy = buf((n, m, h, w), off, g)
    y, dx, dw = empty((n, m, h, w), off), empty((n, k, h, w), off), empty((m, k, 1, 1), off)
    db = empty((m,), off) if bias else None
    op("conv1x1_fwd", [x, wt, b, y, n, k, m, h * w])
    op("conv1x1_bwd", [x, wt, dy, dx, dw, db, n, k, m, h * w])
    R = ref_op("pw", {}, {"x": x.double(), "dy": dy.double(), "w": wt.double(), "bias": b.double() if bias else None})
    checks = [("y", nerr(y, *R["y"])), ("dx", nerr(dx, *R["dx"])), ("dw", nerr(dw, *R["dw"]))]
    if bias:
        checks.append(("db", nerr(db, *R["dbias"])))
    check_all("conv1x1 %s" % (case,), checks)


@pytest.mark.gpu
@pytest.mark.parametrize("case", DW, ids=lambda c: "N%d_C%d_%dx%d_k%d_s%d" % c)
def test_dwconv(case):
    n, c, h, w, ks, s = case
    g = torch.Generator(device="cuda").manual_seed(hash(case) % 2 ** 31)
    x = buf((n, c, h, w), 0, g)
    wt = buf((c, 1, ks, ks), 0, g)
    ho, wo = (h + 2 * (ks // 2) - ks) // s + 1, (w + 2 * (ks // 2) - ks) // s + 1
    y = empty((n, c, ho, wo), 0)
    dy = buf((n, c, ho, wo), 0, g)
    dx, dw = empty((n, c, h, w), 0), empty((c, 1, ks, ks), 0)
    op("dwconv_fwd", [x, wt, y, n, c, h, w, ks, s])
    op("dwconv_bwd", [x, wt, dy, dx, dw, n, c, h, w, ks, s])
    R = ref_op("dw", {"ks": ks, "stride": s}, {"x": x.double(), "dy": dy.double(), "w": wt.double()})
    check_all("dwconv %s" % (case,), [("y", nerr(y, *R["y"])), ("dx", nerr(dx, *R["dx"])), ("dw", nerr(dw, *R["dw"]))])


@pytest.mark.gpu
@pytest.mark.parametrize("case", STEM, ids=lambda c: "N%d_M%d_%dx%d" % c)
def test_stem(case):
    n, m, h, w = case
    g = torch.Generator(device="cuda").manual_seed(hash(case) % 2 ** 31)
    x = torch.rand((n, 3, h, w), device="cuda", generator=g)
    wt = buf((m, 3, 3, 3), 0, g)
    y, dw = empty((n, m, h // 2, w // 2), 0), empty((m, 3, 3, 3), 0)
    dy = buf((n, m, h // 2, w // 2), 0, g)
    op("stem_fwd", [x, wt, y, n, m, h, w])
    op("stem_wgrad", [x, dy, dw, n, m, h, w])
    R = ref_op("stem", {}, {"x": x.double(), "dy": dy.double(), "w": wt.double()})
    check_all("stem %s" % (case,), [("y", nerr(y, *R["y"])), ("dw", nerr(dw, *R["dw"]))])


def bn_run(x, gamma, beta, rm, rv, relu, dy, off=0):
    n, c, h, w = x.shape
    y, dx = empty(x.shape, off), empty(x.shape, off)
    mean, inv = empty((c,), 0), empty((c,), 0)
    dg, db = empty((c,), 0), empty((c,), 0)
    scr = torch.empty(2 * c, dtype=torch.float64, device="cuda")
    op("bn_train_fwd", [x, gamma, beta, rm, rv, y, mean, inv, scr, n, c, h * w, int(relu)])
    op("bn_train_bwd", [x, y, dy, gamma, mean, inv, dx, dg, db, scr, n, c, h * w, int(relu)])
    return y, mean, inv, dx, dg, db


@pytest.mark.gpu
@pytest.mark.parametrize("case", BN, ids=lambda c: "N%d_C%d_%dx%d%s_mean%g%s" % (c[0], c[1], c[2], c[3], "_relu" if c[4] else "", c[5], "_off%d" % c[7] if c[7] else ""))
def test_bn_train(case):
    n, c, h, w, relu, mu, spread, off = case
    g = torch.Generator(device="cuda").manual_seed(hash(case) % 2 ** 31)
    x = buf((n, c, h, w), off, g, spread, mu)
    gamma = torch.rand(c, device="cuda", generator=g) + 0.5
    beta = torch.randn(c, device="cuda", generator=g) * 0.3
    rm, rv = torch.randn(c, device="cuda", generator=g), torch.rand(c, device="cuda", generator=g) + 0.5
    rm0, rv0 = rm.double(), rv.double()
    dy = buf((n, c, h, w), off, g)
    y, mean, inv, dx, dg, db = bn_run(x, gamma, beta, rm, rv, relu, dy, off)
    t = {"x": x.double(), "dy": dy.double(), "y": y.double(), "gamma": gamma.double(), "beta": beta.double(), "mean": mean.double(),
         "invstd": inv.double()}
    R = ref_op("bn", {"relu": relu}, t)
    checks = [("y", nerr(y, *R["y"])), ("mean", nerr(mean, *R["mean"])), ("invstd", nerr(inv, *R["invstd"])),
              ("running_mean", nerr(rm, 0.9 * rm0 + 0.1 * R["mean"][0], 0.9 * rm0.abs() + 0.1 * R["mean"][1])),
              ("running_var", nerr(rv, 0.9 * rv0 + 0.1 * R["var_unbiased"][0], 0.9 * rv0.abs() + 0.1 * R["var_unbiased"][1])),
              ("dx", nerr(dx, *R["dx"])), ("dgamma", nerr(dg, *R["dgamma"])), ("dbeta", nerr(db, *R["dbeta"]))]
    check_all("bn %s" % (case,), checks)


@pytest.mark.gpu
@pytest.mark.parametrize("case", POOL, ids=lambda c: "N%d_C%d_%dx%d" % c)
def test_maxpool(case):
    n, c, h, w = case
    g = torch.Generator(device="cuda").manual_seed(hash(case) % 2 ** 31)
    x = torch.randn((n, c, h, w), device="cuda", generator=g).relu_()          # ReLU output: exact ties at 0
    pool_against_torch(x)


@pytest.mark.gpu
@pytest.mark.parametrize("case", UP, ids=lambda c: "N%d_C%d_%dx%d" % c)
def test_upsample(case):
    n, c, h, w = case
    g = torch.Generator(device="cuda").manual_seed(hash(case) % 2 ** 31)
    x = torch.randn((n, c, h, w), device="cuda", generator=g)
    y = empty((n, c, 2 * h, 2 * w), 0)
    dy = torch.randn(y.shape, device="cuda", generator=g)
    dx = empty(x.shape, 0)
    op("upsample2_fwd", [x, y, n * c, h, w])
    op("upsample2_bwd", [dy, dx, n * c, h, w])
    assert torch.equal(y, F.interpolate(x, scale_factor=2))
    R = ref_op("up", {}, {"x": x.double(), "dy": dy.double()})
    check_all("upsample %s" % (case,), [("dx", nerr(dx, *R["dx"]))])


def pool_against_torch(x):
    """values, indices and the backward of our max-pool equal torch CUDA's max_pool2d (NaN where torch has NaN)"""
    n, c, h, w = x.shape
    ho, wo = (h - 1) // 2 + 1, (w - 1) // 2 + 1
    y, idx = empty((n, c, ho, wo), 0), torch.empty((n, c, ho, wo), dtype=torch.int32, device="cuda")
    op("maxpool_fwd", [x, y, idx, n * c, h, w])
    xr = x.clone().requires_grad_(True)
    yt, it = F.max_pool2d(xr, 3, 2, 1, return_indices=True)
    torch.testing.assert_close(y, yt.detach(), rtol=0, atol=0, equal_nan=True)
    assert torch.equal(idx.long(), it), (idx, it)
    dy = torch.randn(y.shape, device="cuda")
    dx = empty(x.shape, 0)
    op("maxpool_bwd", [dy, idx, dx, n * c, h, w])
    yt.backward(dy)
    torch.testing.assert_close(dx, xr.grad, rtol=1e-6, atol=1e-6, equal_nan=True)


# ---- special values ------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_maxpool_nan_inf_and_ties_like_torch():
    """ATen keeps the first maximum but lets a NaN always win, so a window holding NaNs reports the last of them; +-inf, exact ties,
    all-equal and all -inf windows keep the first position."""
    nan, inf = float("nan"), float("inf")
    x = torch.zeros(1, 6, 5, 6, device="cuda")
    x[0, 0, :3, :3] = torch.tensor([[1, nan, 3], [nan, 0, 0], [2, 2, 2]])            # the window of output (1, 1) holds both NaNs
    x[0, 1] = torch.arange(30, device="cuda").view(5, 6).float()
    x[0, 1, 2, 2] = nan
    x[0, 2] = 7.0                                                                      # all-equal windows
    x[0, 3] = -inf                                                                     # all -inf
    x[0, 3, 4, 5] = inf
    x[0, 4] = torch.tensor([[0, 5, 5, 1, 5, 0]] * 5, device="cuda").float()           # ties across window edges
    x[0, 5, 1, :] = torch.tensor([-inf, nan, inf, nan, 3, -inf])
    pool_against_torch(x)
    x = torch.tensor([[[[1, nan, 3], [nan, 0, 0], [2, 2, 2]]]], device="cuda")
    y, idx = empty((1, 1, 2, 2), 0), torch.empty((1, 1, 2, 2), dtype=torch.int32, device="cuda")
    op("maxpool_fwd", [x, y, idx, 1, 3, 3])
    assert torch.isnan(y[0, 0, 0, 0]) and int(idx[0, 0, 0, 0]) == 3                    # the window [[1, nan], [nan, 0]]: its last NaN
    pool_against_torch(x)


def bn_relu_torch(x, gamma, beta, dy):
    xr, gr, br = x.clone().requires_grad_(True), gamma.clone().requires_grad_(True), beta.clone().requires_grad_(True)
    y = F.relu(F.batch_norm(xr, None, None, gr, br, True, 0.1, 1e-5))
    y.backward(dy)
    return y.detach(), xr.grad, gr.grad, br.grad


@pytest.mark.gpu
@pytest.mark.parametrize("special", ["nan", "inf", "-inf", "constant"])
def test_bn_relu_special_values_like_torch(special):
    """BatchNorm + ReLU where a channel holds a NaN or an infinity (its statistics become NaN: torch's ReLU keeps NaN, where fmaxf
    would return 0) or is constant (variance 0, y = beta, exact ties of ReLU at 0 when beta <= 0); values where torch has NaN must be
    NaN, the rest within the fp32 reference's tolerance."""
    g = torch.Generator(device="cuda").manual_seed(7)
    x = torch.randn(3, 4, 5, 6, device="cuda", generator=g)
    if special == "constant":
        x[:, 1] = 2.5
        x[:, 2] = -1.0
    else:
        x[1, 2, 3, 4] = float(special)
    gamma = torch.tensor([1.0, 0.7, 1.3, 0.9], device="cuda")
    beta = torch.tensor([0.1, -0.2, 0.0, 0.3], device="cuda")
    dy = torch.randn(x.shape, device="cuda", generator=g)
    y, _, _, dx, dg, db = bn_run(x, gamma, beta, torch.zeros(4, device="cuda"), torch.ones(4, device="cuda"), True, dy)
    yt, dxt, dgt, dbt = bn_relu_torch(x, gamma, beta, dy)
    for name, a, b in (("y", y, yt), ("dx", dx, dxt), ("dgamma", dg, dgt), ("dbeta", db, dbt)):
        assert torch.equal(torch.isnan(a), torch.isnan(b)), (name, torch.isnan(a).sum().item(), torch.isnan(b).sum().item())
        torch.testing.assert_close(a, b, rtol=1e-4, atol=1e-4, equal_nan=True, msg=name)
    if special != "constant":
        assert torch.isnan(y[:, 2]).all() and not torch.isnan(y[:, [0, 1, 3]]).any()


@pytest.mark.gpu
@pytest.mark.parametrize("pyops", [False, True], ids=["native", "pyops"])
def test_one_value_per_channel_is_refused_like_torch(pyops, monkeypatch):
    """N = 1 at 32x32: every stride-32 BatchNorm would normalise one value.  The reference's F.batch_norm raises ValueError; so do
    both training paths, before anything is launched (the running statistics stay untouched)."""
    import model.detector as det
    import synth
    if pyops:
        from model import train_ops
        monkeypatch.setattr(train_ops, "forward_train_native", train_ops.forward_train)
    m = det.Detector(80, 3, True)
    m.load_state_dict(synth.make_state_dict(5), strict=True)
    m = m.cuda().train()
    before = [t.clone() for t in m.state_dict().values()]
    x = synth.make_images(6, 1, 32, 32).cuda()
    with pytest.raises(ValueError, match="Expected more than 1 value per channel when training"):
        m(x)
    assert all(torch.equal(a, b) for a, b in zip(before, m.state_dict().values()))
    with pytest.raises(ValueError, match="Expected more than 1 value per channel when training"):
        F.batch_norm(torch.ones(1, 96, 1, 1, device="cuda"), None, None, training=True)
    m(synth.make_images(6, 1, 32, 64).cuda())                                          # two values per channel: accepted
