"""Which kernel variants (cells) the training operators (csrc/k_train.cu) and the native trainer's step (csrc/trainer.cu) reach,
read from the library's own launch records (yfv2_op_debug_launches / yfv2_trainer_debug_launches), and an independent statement of
the trainer's program.

A *cell* is one (site, variant) pair, e.g. ("wgrad", "rows / partial / multi-chunk") or ("bn_stats", "float4"): the dispatch cells
come from the records (kernel, tile height, float4 choices, pixel chunks, partial sums, BatchNorm slices, grids), the input-shape
cells (maps smaller than the stencil, odd inputs, ReLU, bias, ...) from the op's shapes.  op_cells() gives the cells of one
yfv2_op_* call, trainer_cells() those of one training step of a library trainer at (N, H, W, A, C); `find_case()` searches
trainer shapes for one that reaches a given cell.  tests/test_train_dispatch_cpu.py pins `program()` against the trainer's own op
list (yfv2_trainer_debug_ops) and checks that the case lists of tests/test_train_fp64_gpu.py and tests/test_train_ops_space_gpu.py
reach every cell."""
import ctypes
import functools

STAGE_REPEATS = (4, 8, 4)            # trainer.cu kStageRepeats
STAGE_OUT = (48, 96, 192)            # trainer.cu kStageOut


# ---- cells of launch records --------------------------------------------------------------------------------------------------
def bucket_slices(s):
    return "1" if s == 1 else "64 (cap)" if s == 64 else "2..63"


def shape_cells(kind, s):
    """The input-shape cells of one op: kind as yfv2_trainer_op.kind, s = dict(N, C, H, W) of its input (+ M, ks, stride, relu,
    bias where the op has them)."""
    out = set()
    if kind == "pw" and s["bias"]:
        out.add(("conv1x1", "bias"))
    elif kind == "dw":
        ks, st = s["ks"], s["stride"]
        out.add(("dw", "%dx%d s%d" % (ks, ks, st)))
        if s["H"] < ks or s["W"] < ks:
            out.add(("dw", "map smaller than the stencil"))
        if st == 2 and (s["H"] % 2 or s["W"] % 2):
            out.add(("dw", "s2 odd input"))
    elif kind == "bn":
        out.add(("bn", "relu" if s["relu"] else "no relu"))
        if s["N"] * s["H"] * s["W"] == 2:
            out.add(("bn", "2 values per channel"))
    elif kind == "stem":
        out.add(("stem_wgrad", "M%4=0" if s["M"] % 4 == 0 else "M%4!=0"))
    elif kind == "pool":
        out.add(("maxpool", "odd input" if s["H"] % 2 or s["W"] % 2 else "even input"))
    return out


def record_cells(r, s):
    """The dispatch cells of one launch record r (a dict of yfv2_engine's TrainLaunchRecord) of an op whose input is s."""
    k = r["kernel"]
    hw = s["H"] * s["W"]
    vec = lambda v: "float4" if v else "scalar"
    if k.startswith("gemm2_kernel"):
        why = "scalar: HW%4" if hw % 4 else "scalar: unaligned"
        return {("gemm2", "BM=%d" % r["bm"]), ("gemm2 B", "float4" if r["vec_b"] else why), ("gemm2 C", "float4" if r["vec_c"] else why)}
    if k.startswith(("wgrad_rows_kernel", "wgrad1x1_kernel")):
        kern = "rows" if k.startswith("wgrad_rows") else "tiled" + k[k.index("<") + 1:-1]
        out = {("wgrad", "%s / %s / %s" % (kern, "partial" if r["partial"] else "atomic", "multi-chunk" if r["chunks"] > 1 else "one chunk"))}
        if kern == "rows" and r["grid"][1] > 1:
            out.add(("wgrad", "rows / blockIdx.y > 0"))
        return out
    if k.startswith("dw_wgrad_kernel"):
        return {("dw_wgrad", "batch loop (N > 16)" if r["grid"][1] < s["N"] else "grid.y = N")}
    if k == "bn_stats_kernel":
        return {("bn_stats", vec(r["vec"])), ("bn slices", bucket_slices(r["slices"]))}
    if k == "bn_apply_kernel":
        return {("bn_apply", vec(r["vec"])), ("bn y-grid", ">1" if r["grid"][1] > 1 else "1")}
    if k.startswith("stem_fwd"):
        return {("stem_fwd", "stem_fwd_kernel<24>" if k == "stem_fwd_kernel<24>" else "generic")}
    if k == "upsample2_fwd_kernel":
        return {("upsample", "2x")}
    if k == "chan_copy_kernel":
        return {("chan_copy", "accumulate" if r["accumulate"] else "assign")}
    return set()


def op_cells(name, ptrs, ints, sms):
    """The cells one yfv2_op_<name> call reaches (ptrs: integer addresses or None, ints: its integer arguments)."""
    import yfv2_engine
    if name.startswith("conv1x1"):
        n, k, m, hw = ints
        s = dict(N=n, C=k, H=hw, W=1, M=m, bias=ptrs[2 if name == "conv1x1_fwd" else 5] is not None)
        kind = "pw"
    elif name.startswith("dwconv"):
        s = dict(zip(("N", "C", "H", "W", "ks", "stride"), ints))
        kind = "dw"
    elif name.startswith("stem"):
        s = dict(zip(("N", "M", "H", "W"), ints))
        kind = "stem"
    elif name.startswith("bn"):
        s = dict(zip(("N", "C", "H", "relu"), ints), W=1)
        kind = "bn"
    else:
        s = dict(zip(("N", "H", "W"), ints))
        kind = "pool" if name.startswith("maxpool") else "up"
    out = shape_cells(kind, s)
    for r in yfv2_engine.op_launches(name, ptrs, ints, sms):
        out |= record_cells(r, s)
    return out


# ---- the trainer's program (trainer.cu build()) -------------------------------------------------------------------------------
KIND = ("stem", "bn", "pool", "pw", "dw", "up", "odd", "cate", "cat2")             # trainer.cu enum Kind


@functools.lru_cache(maxsize=None)
def program(N, H, W, A=3, C=80):
    """(ops, tensors, pnumel): the trainer's op list in forward order with the fields of yfv2_trainer_op (aux omitted), every
    tensor's (C, H, W, ext) and every parameter's numel, as trainer.cu build() lays them out."""
    pnumel, tens, ops = [], [], []
    nbn = [0]

    def param(n):
        pnumel.append(n)
        return len(pnumel) - 1

    def conv_bn(wn, c):
        i = param(wn); param(c); param(c)
        nbn[0] += 1
        return (i, i + 1, i + 2, nbn[0] - 1)

    def ten(c, h, w, ext=-1):
        tens.append((c, h, w, ext))
        return len(tens) - 1

    def push(kind, a, y, b=-1, pw=-1, pg=-1, pb=-1, pbias=-1, bn=-1, relu=0, ks=0, stride=0, M=0):
        ops.append(dict(kind=kind, a=a, b=b, y=y, pw=pw, pg=pg, pb=pb, pbias=pbias, bn=bn, relu=relu, ks=ks, stride=stride, M=M))
        return y

    def bnop(x, cb, relu):
        c, h, w, _ = tens[x]
        return push("bn", x, ten(c, h, w), pg=cb[1], pb=cb[2], bn=cb[3], relu=int(relu))

    def pwop(x, w, m, bias=-1, ext=-1):
        _, h, ww, _ = tens[x]
        return push("pw", x, ten(m, h, ww, ext), pw=w, pbias=bias, M=m)

    def dwop(x, w, ks, s):
        c, h, ww, _ = tens[x]
        return push("dw", x, ten(c, (h + 2 * (ks // 2) - ks) // s + 1, (ww + 2 * (ks // 2) - ks) // s + 1), pw=w, ks=ks, stride=s)

    pw_bn = lambda x, cb, m, relu: bnop(pwop(x, cb[0], m), cb, relu)
    dw_bn = lambda x, cb, ks, s, relu: bnop(dwop(x, cb[0], ks, s), cb, relu)

    first = conv_bn(24 * 27, 24)
    blk, cin = [], 24
    for st in range(3):
        K = STAGE_OUT[st] // 2
        for r in range(STAGE_REPEATS[st]):
            s = 2 if r == 0 else 1
            q = dict(K=K, stride=s, pw1=conv_bn(K * (cin if s == 2 else K), K), dw=conv_bn(K * 9, K), pw2=conv_bn(K * K, K))
            if s == 2:
                q["pdw"] = conv_bn(cin * 9, cin); q["ppw"] = conv_bn(K * cin, K)
            blk.append(q)
        cin = STAGE_OUT[st]
    c2, c3 = conv_bn(72 * 288, 72), conv_bn(72 * 192, 72)
    head = [[conv_bn(72 * 25, 72), conv_bn(72 * 72, 72), conv_bn(72 * 25, 72), conv_bn(72 * 72, 72)] for _ in range(4)]
    w_reg = param(4 * A * 72); b_reg = param(4 * A)
    w_obj = param(A * 72); b_obj = param(A)
    w_cls = param(C * 72); b_cls = param(C)

    xin = ten(3, H, W, -2)
    x = push("stem", xin, ten(24, H // 2, W // 2), pw=first[0])
    x = bnop(x, first, True)
    _, h, w, _ = tens[x]
    x = push("pool", x, ten(24, (h - 1) // 2 + 1, (w - 1) // 2 + 1))
    feat = []
    for st in range(3):
        for r in range(STAGE_REPEATS[st]):
            q = blk[sum(STAGE_REPEATS[:st]) + r]
            K = q["K"]
            if q["stride"] == 2:
                proj = pw_bn(dw_bn(x, q["pdw"], 3, 2, False), q["ppw"], K, True)
                m = pw_bn(x, q["pw1"], K, True)
                m = dw_bn(m, q["dw"], 3, 2, False)
                m = pw_bn(m, q["pw2"], K, True)
                x = push("cat2", proj, ten(2 * K, tens[m][1], tens[m][2]), b=m)
            else:
                m = push("odd", x, ten(K, tens[x][1], tens[x][2]))
                m = pw_bn(m, q["pw1"], K, True)
                m = dw_bn(m, q["dw"], 3, 1, False)
                m = pw_bn(m, q["pw2"], K, True)
                x = push("cate", x, ten(2 * K, tens[m][1], tens[m][2]), b=m)
        feat.append(x)
    C2, C3 = feat[1], feat[2]
    S3 = pw_bn(C3, c3, 72, True)

    def run_head(hd, s):
        y = dw_bn(s, hd[0], 5, 1, True)
        y = pw_bn(y, hd[1], 72, False)
        y = dw_bn(y, hd[2], 5, 1, True)
        return pw_bn(y, hd[3], 72, False)

    cls3, reg3 = run_head(head[3], S3), run_head(head[2], S3)
    up = push("up", C3, ten(192, 2 * tens[C3][1], 2 * tens[C3][2]))
    P2 = push("cat2", up, ten(288, tens[C2][1], tens[C2][2]), b=C2)
    S2 = pw_bn(P2, c2, 72, True)
    cls2, reg2 = run_head(head[0], S2), run_head(head[1], S2)
    for lv, (cl, rg) in enumerate(((cls2, reg2), (cls3, reg3))):
        pwop(rg, w_reg, 4 * A, b_reg, 3 * lv)
        pwop(cl, w_obj, A, b_obj, 3 * lv + 1)
        pwop(cl, w_cls, C, b_cls, 3 * lv + 2)
    return tuple(ops), tuple(tens), tuple(pnumel)


def consumers(ops, ntens):
    """tensor id -> op indices that read it, in forward order"""
    out = [[] for _ in range(ntens)]
    for i, o in enumerate(ops):
        for t in (o["a"], o["b"]):
            if t >= 0:
                out[t].append(i)
    return out


def pscratch_floats(pnumel, A, C):
    """trainer.cu build(): the parameter-gradient scratch holds the largest parameter and weight + bias of each shared output conv"""
    n = len(pnumel)
    return max(max(pnumel), *(pnumel[i] + pnumel[i + 1] for i in (n - 6, n - 4, n - 2)))


def trainer_cells(N, H, W, A=3, C=80, sms=132):
    """The cells one training step (forward + backward) of a library trainer at (N, H, W, A, C) reaches, from its launch records."""
    import yfv2_engine
    lib = yfv2_engine.lib()
    t = ctypes.c_void_p()
    yfv2_engine._check(lib.yfv2_trainer_create(ctypes.byref(t), 0, N, H, W, A, C), "trainer_create")
    try:
        ops, tens, layout = yfv2_engine.trainer_program(t)
        recs = yfv2_engine.trainer_launches(t, sms=sms)
    finally:
        lib.yfv2_trainer_destroy(t)
    shapes = []
    for o in ops:
        x = tens[o["a"]]
        shapes.append(dict(N=N, C=x["C"], H=x["H"], W=x["W"], M=tens[o["y"]]["C"], ks=o["ks"], stride=o["stride"], relu=o["relu"],
                           bias=o["pbias"] >= 0))
    out = set()
    for o, s in zip(ops, shapes):
        out |= shape_cells(o["kind"], s)
    for r in recs:
        if r["op"] >= 0:
            out |= record_cells(r, shapes[r["op"]])
    # the trainer's accumulation structure: a tensor read by several ops (not an odd / cate pair) sums their gradients through the
    # scratch tensor; the shared output convolutions' second use goes through the parameter scratch
    for t_, cs in enumerate(consumers(ops, len(tens))):
        if len(cs) > 1 and not any(ops[j]["kind"] in ("odd", "cate") for j in cs):
            out.add(("fan-in", "scratch + axpy"))
    out.add(("pscratch", "shared output conv"))
    if layout["pscratch_floats"] > max(program(N, H, W, A, C)[2]):
        out.add(("pscratch", "weight + bias above every parameter"))
    return out


# ---- every cell, and where each can be reached -----------------------------------------------------------------------------
ALL_CELLS = frozenset(
    [("gemm2", "BM=32"), ("gemm2", "BM=64")]
    + [(s, v) for s in ("gemm2 B", "gemm2 C") for v in ("float4", "scalar: HW%4", "scalar: unaligned")]
    + [("wgrad", "%s / %s / %s" % (k, p, c)) for k in ("rows", "tiled32", "tiled64") for p in ("partial", "atomic")
       for c in ("one chunk", "multi-chunk")]
    + [("wgrad", "rows / blockIdx.y > 0"), ("conv1x1", "bias")]
    + [("dw", "%dx%d s%d" % (k, k, s)) for k in (3, 5) for s in (1, 2)]
    + [("dw", "map smaller than the stencil"), ("dw", "s2 odd input"), ("dw_wgrad", "grid.y = N"), ("dw_wgrad", "batch loop (N > 16)")]
    + [(s, v) for s in ("bn_stats", "bn_apply") for v in ("float4", "scalar")]
    + [("bn slices", v) for v in ("1", "2..63", "64 (cap)")] + [("bn y-grid", "1"), ("bn y-grid", ">1")]
    + [("bn", "relu"), ("bn", "no relu"), ("bn", "2 values per channel")]
    + [("stem_fwd", "stem_fwd_kernel<24>"), ("stem_fwd", "generic"), ("stem_wgrad", "M%4=0"), ("stem_wgrad", "M%4!=0")]
    + [("maxpool", "even input"), ("maxpool", "odd input"), ("upsample", "2x")]
    # (a concat's backward never accumulates: each of its inputs is read last by the concat itself, so it runs first and assigns)
    + [("chan_copy", "assign"), ("fan-in", "scratch + axpy")]
    + [("pscratch", "shared output conv"), ("pscratch", "weight + bias above every parameter")])

# cells only the trainer reaches: the op ABI passes no weight-gradient scratch (so never the partial path) and has no program
TRAINER_ONLY = frozenset(c for c in ALL_CELLS if c[0] in ("chan_copy", "fan-in", "pscratch") or "partial" in c[1])

SEARCH_SIDES = (32, 64, 96, 128, 192, 256, 352, 512, 544, 640)
SEARCH_BATCHES = (1, 2, 3, 4, 8, 16, 32, 64, 102, 128, 203, 256)
SEARCH_HEADS = ((3, 80), (3, 300))


@functools.lru_cache(maxsize=None)
def reachable(sms=132):
    """cell -> the cheapest (fewest input pixels) trainer case (n, h, w, a, c) of the search space that reaches it"""
    best = {}
    for h in SEARCH_SIDES:
        for w in SEARCH_SIDES:
            for n in SEARCH_BATCHES:
                if n * (h // 32) * (w // 32) == 1:                                   # refused: BatchNorm over one value
                    continue
                for a, c in SEARCH_HEADS:
                    cost = (n * h * w, c)
                    for cl in trainer_cells(n, h, w, a, c, sms):
                        if cl not in best or cost < best[cl][0]:
                            best[cl] = (cost, (n, h, w, a, c))
    return {cl: v[1] for cl, v in best.items()}


def find_case(cell, sms=132):
    """The cheapest trainer case (n, h, w, a, c) of the search space whose training step reaches `cell`, or None."""
    return reachable(sms).get(cell)
