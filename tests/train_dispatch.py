"""Python model of the host choices of the training kernels (csrc/k_train.cu) and of the native trainer's program
(csrc/trainer.cu).

Every rule below restates the C++ source named beside it.  A *cell* is one (operator, variant) pair, e.g. ("wgrad", "rows /
partial / multi-chunk") or ("bn_stats", "float4"); pw_cells() / dw_cells() / bn_cells() / stem_cells() / pool_cells() give the
cells one yfv2_op_* call reaches, trainer_cells() the cells a training step of the native trainer at (N, H, W, A, C) reaches.  `find_case()` searches trainer shapes for one that reaches
a given cell.  tests/test_train_dispatch_cpu.py pins `program()` against the trainer's own op list (yfv2_trainer_debug_ops) and
checks that the case lists of tests/test_train_fp64_gpu.py and tests/test_train_ops_space_gpu.py reach every cell."""
import functools

K_WSCRATCH_FLOATS = 4 << 20          # trainer.cu kWScratchFloats: per-block weight-gradient partials of one layer
STAGE_REPEATS = (4, 8, 4)            # trainer.cu kStageRepeats
STAGE_OUT = (48, 96, 192)            # trainer.cu kStageOut


# ---- k_train.cu host rules --------------------------------------------------------------------------------------------------
def gemm2(M, N, sB, sC, b_aligned=True, c_aligned=True):
    """run_gemm2 / gemm2_kernel: the tile height and the float4 conditions of B and C.  sB = (sBk, sBb), sC = (sCi, sCb)."""
    bm = 32 if M <= 32 else 64                                                       # run_gemm2: g.M <= 32
    vec_b = N % 4 == 0 and all(s % 4 == 0 for s in sB) and b_aligned                 # gemm2_kernel vecB (B 16-byte aligned)
    vec_c = N % 4 == 0 and all(s % 4 == 0 for s in sC) and c_aligned                 # gemm2_kernel vecC
    return bm, vec_b, vec_c


def gemm2_variant(vec, hw):
    return "float4" if vec else "scalar: HW%4" if hw % 4 else "scalar: unaligned"


def wgrad(N, K, M, HW, sms, scratch_floats=0, tiled_only=False):
    """conv1x1_bwd_impl's weight-gradient choice: (kernel, pchunk, chunks, partial, row groups)."""
    if K == 24 and M % 24 == 0 and not tiled_only:                                   # wgrad_rows_kernel<24, 3>
        pchunk = 2048
        while pchunk > 256 and N * (M // 24) * -(-HW // pchunk) < 2 * sms:
            pchunk >>= 1
        kern, groups = "rows", M // 24
    else:
        bt = 32 if M <= 32 and K <= 32 else 64                                       # wgrad1x1_kernel<BT>
        tiles = -(-M // bt) * -(-K // bt)
        pchunk = 1024
        while pchunk > 64 and tiles * N * -(-HW // pchunk) < 4 * sms:
            pchunk >>= 1
        kern, groups = "tiled%d" % bt, 1
    chunks = -(-HW // pchunk)
    partial = scratch_floats > 0 and N * chunks * M * K <= scratch_floats           # else memset + fp32 atomics
    return kern, pchunk, chunks, partial, groups


def bn_slices(N, HW):                                                                # yfv2_op_bn_train_fwd / _bwd
    s = -(-(N * HW) // (256 * 16))
    s = min(max(s, 1), 64)
    return min(s, N)


def bucket_slices(s):
    return "1" if s == 1 else "64 (cap)" if s == 64 else "2..63"


# ---- cells of one op call -----------------------------------------------------------------------------------------------------
def pw_cells(N, K, M, HW, sms, bias=False, scratch_floats=0, x_aligned=True, y_aligned=True, dx=True, tiled_only=False):
    """yfv2_op_conv1x1_fwd + conv1x1_bwd_impl: x [N,K,HW] -> y [N,M,HW]."""
    out = set()
    bm, vb, vc = gemm2(M, HW, (HW, K * HW), (HW, M * HW), x_aligned, y_aligned)      # forward: B = x, C = y
    out |= {("gemm2", "BM=%d" % bm), ("gemm2 B", gemm2_variant(vb, HW)), ("gemm2 C", gemm2_variant(vc, HW))}
    if dx:
        bm, vb, vc = gemm2(K, HW, (HW, M * HW), (HW, K * HW), y_aligned, x_aligned)  # dgrad: B = dy, C = dx
        out |= {("gemm2", "BM=%d" % bm), ("gemm2 B", gemm2_variant(vb, HW)), ("gemm2 C", gemm2_variant(vc, HW))}
    kern, _, chunks, partial, groups = wgrad(N, K, M, HW, sms, scratch_floats, tiled_only)
    out.add(("wgrad", "%s / %s / %s" % (kern, "partial" if partial else "atomic", "multi-chunk" if chunks > 1 else "one chunk")))
    if kern == "rows" and groups > 1:
        out.add(("wgrad", "rows / blockIdx.y > 0"))
    if bias:
        out.add(("conv1x1", "bias"))
    return out


def dw_cells(N, C, H, W, ks, stride):
    out = {("dw", "%dx%d s%d" % (ks, ks, stride))}
    if H < ks or W < ks:
        out.add(("dw", "map smaller than the stencil"))
    if stride == 2 and (H % 2 or W % 2):
        out.add(("dw", "s2 odd input"))
    out.add(("dw_wgrad", "batch loop (N > 16)" if N > 16 else "grid.y = N"))
    return out


def bn_cells(N, C, HW, relu, aligned=True):
    vec = HW % 4 == 0 and aligned
    out = {("bn_stats", "float4" if vec else "scalar"), ("bn_apply", "float4" if vec else "scalar"),
           ("bn slices", bucket_slices(bn_slices(N, HW))), ("bn y-grid", ">1" if HW > 1024 else "1"),
           ("bn", "relu" if relu else "no relu")}
    if N * HW == 2:
        out.add(("bn", "2 values per channel"))
    return out


def stem_cells(N, M, H, W):
    return {("stem_fwd", "stem_fwd_kernel<24>" if M == 24 else "generic"), ("stem_wgrad", "M%4=0" if M % 4 == 0 else "M%4!=0")}


def pool_cells(H, W):
    return {("maxpool", "odd input" if H % 2 or W % 2 else "even input")}


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
    """The cells one training step (forward + backward) of the native trainer reaches."""
    ops, tens, pnumel = program(N, H, W, A, C)
    cons = consumers(ops, len(tens))
    out = set()
    for i, o in enumerate(ops):
        c, h, w, _ = tens[o["a"]]
        k = o["kind"]
        if k == "stem":
            out |= stem_cells(N, tens[o["y"]][0], h, w)
        elif k == "bn":
            out |= bn_cells(N, c, h * w, o["relu"])
        elif k == "pool":
            out |= pool_cells(h, w)
        elif k == "pw":
            out |= pw_cells(N, c, o["M"], h * w, sms, o["pbias"] >= 0, K_WSCRATCH_FLOATS)
        elif k == "dw":
            out |= dw_cells(N, c, h, w, o["ks"], o["stride"])
        elif k == "up":
            out.add(("upsample", "2x"))
        elif k in ("odd", "cate"):
            out.add(("chan_copy", "assign"))
        elif k == "cat2":
            acc = any(cons[t][-1] != i for t in (o["a"], o["b"]))                  # run_backward: not the tensor's last use
            out.add(("chan_copy", "accumulate" if acc else "assign"))
    for t, cs in enumerate(cons):
        if len(cs) > 1 and not any(ops[j]["kind"] in ("odd", "cate") for j in cs):
            out.add(("fan-in", "scratch + axpy"))
    out.add(("pscratch", "shared output conv"))
    if pscratch_floats(pnumel, A, C) > max(pnumel):
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
