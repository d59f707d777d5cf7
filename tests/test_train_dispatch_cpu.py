"""CPU: the trainer's program (tests/train_dispatch.py) against the native trainer's own, read through the host-only hooks
yfv2_trainer_debug_ops / _tensors / _layout; the case lists of the fp64 training suites against every cell the library's launch
records reach; the records on both sides of each dispatch rule; and the refusals that need no device."""
import ctypes

import pytest

import yfv2  # noqa: F401
import train_dispatch as td

SHAPES = [(2, 32, 32, 3, 80), (1, 32, 64, 3, 80), (3, 64, 96, 2, 20), (2, 640, 352, 3, 80), (64, 352, 352, 3, 300)]


def trainer(N, H, W, A, C):
    import yfv2_engine
    lib = yfv2_engine.lib()
    t = ctypes.c_void_p()
    assert lib.yfv2_trainer_create(ctypes.byref(t), 0, N, H, W, A, C) == 0, lib.yfv2_last_error()
    return lib, t


@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "%dx%dx%d_a%d_c%d" % s)
def test_program_matches_the_trainer(shape):
    import yfv2_engine
    lib, t = trainer(*shape)
    try:
        ops, tens, layout = yfv2_engine.trainer_program(t)
        mops, mtens, pnumel = td.program(*shape)
        assert len(ops) == len(mops)
        for i, (o, mo) in enumerate(zip(ops, mops)):
            assert {k: o[k] for k in mo} == mo, i
            assert (o["aux"] >= 0) == (o["kind"] in ("bn", "pool")), i
        assert [(x["C"], x["H"], x["W"], x["ext"]) for x in tens] == list(mtens)
        N = shape[0]
        # every workspace tensor lies inside the workspace and no two overlap
        spans = sorted((x[k], x[k] + N * x["C"] * x["H"] * x["W"]) for x in tens if x["ext"] == -1 for k in ("off", "goff"))
        spans += [(o["aux"], o["aux"] + (6 * tens[o["a"]]["C"] if o["kind"] == "bn" else N * tens[o["y"]]["C"] * tens[o["y"]]["H"] * tens[o["y"]]["W"]))
                  for o in ops if o["aux"] >= 0]
        spans += [(layout[k + "_off"], layout[k + "_off"] + n) for k, n in
                  (("scratch", max(N * x["C"] * x["H"] * x["W"] for x in tens if x["ext"] == -1)), ("pscratch", layout["pscratch_floats"]),
                   ("gflat", layout["gflat_floats"]), ("wscratch", layout["wscratch_floats"]))]
        spans.sort()
        assert spans[0][0] >= 0 and spans[-1][1] <= layout["ws_floats"]
        assert all(a[1] <= b[0] for a, b in zip(spans, spans[1:]))
        assert layout["gflat_floats"] == sum(pnumel) and layout["wscratch_floats"] == 4 << 20
        assert layout["pscratch_floats"] == td.pscratch_floats(pnumel, shape[3], shape[4])
    finally:
        lib.yfv2_trainer_destroy(t)


def test_pscratch_holds_weight_and_bias_of_the_shared_output_convs():
    """The second use of a shared output convolution puts its bias gradient right behind the weight's in the parameter scratch: at
    300 classes 72 * 300 + 300 floats, more than the largest parameter (72 * 288), and the scratch must hold them."""
    import yfv2_engine
    lib, t = trainer(2, 64, 64, 3, 300)
    try:
        _, _, layout = yfv2_engine.trainer_program(t)
        assert layout["pscratch_floats"] == 73 * 300 > 72 * 288
        assert layout["pscratch_off"] + 73 * 300 <= layout["gflat_off"]
    finally:
        lib.yfv2_trainer_destroy(t)


def test_cases_cover_every_cell():
    """At 132 SMs (H100 SXM): the trainer cases of test_train_fp64_gpu.py reach every cell only a training step can reach, and
    together with the op calls of test_train_ops_space_gpu.py every cell any of the two can reach.  Only the partial-sum path of
    the 32-wide tiled wgrad is reached by neither: the trainer never runs it (its layers of at most 32 channels have 24 inputs and
    take the rows kernel) and the op entry points pass no scratch."""
    import test_train_fp64_gpu as tf
    import test_train_ops_space_gpu as sp
    reach = set(td.reachable(132))
    assert td.ALL_CELLS - reach - (td.ALL_CELLS - td.TRAINER_ONLY) == {("wgrad", "tiled32 / partial / one chunk"),
                                                                     ("wgrad", "tiled32 / partial / multi-chunk")}
    have_tr, have_op = tf.case_cells(132), sp.case_cells(132)
    missing = (reach & td.TRAINER_ONLY) - have_tr
    assert not missing, {cl: td.find_case(cl) for cl in missing}
    missing = (reach | (td.ALL_CELLS - td.TRAINER_ONLY)) - have_tr - have_op
    assert not missing, {cl: td.find_case(cl) for cl in missing}
    assert (have_tr | have_op) <= td.ALL_CELLS


def test_bn_over_one_value_is_refused_before_any_launch():
    import yfv2_engine
    lib = yfv2_engine.lib()
    t = ctypes.c_void_p()
    assert lib.yfv2_trainer_create(ctypes.byref(t), 0, 1, 32, 32, 3, 80) < 0
    assert b"more than 1 value per channel" in lib.yfv2_last_error()
    fake = ctypes.c_void_p(16)                                       # never dereferenced: the refusal comes first
    assert lib.yfv2_op_bn_train_fwd(*[fake] * 9, 1, 8, 1, 1, None) < 0
    assert b"more than 1 value per channel" in lib.yfv2_last_error()
    with pytest.raises(yfv2_engine.Yfv2Error, match="more than 1 value per channel"):
        yfv2_engine.op_launches("bn_train_fwd", [16] * 9, [1, 8, 1, 1])
    with pytest.raises(ValueError, match="Expected more than 1 value per channel when training"):
        yfv2_engine.check_bn_batch(1, 32, 32)
    with pytest.raises(ValueError):
        yfv2_engine.check_bn_batch(1, 30, 20)                      # the op-by-op path's sizes: stride 32 rounds up to 1 x 1
    for n, h, w in ((2, 32, 32), (1, 32, 64), (1, 64, 32), (1, 66, 64)):
        yfv2_engine.check_bn_batch(n, h, w)


# ---- the library's launch records on both sides of each dispatch rule (yfv2_op_debug_launches / yfv2_trainer_debug_launches) ------
A16 = 1 << 20                                                       # a 16-byte-aligned address (never dereferenced)


def recs(name, ptrs, ints, sms=132):
    import yfv2_engine
    return yfv2_engine.op_launches(name, ptrs, ints, sms)


def one(rs, prefix):
    got = [r for r in rs if r["kernel"].startswith(prefix)]
    assert len(got) == 1, [r["kernel"] for r in rs]
    return got[0]


def test_gemm_tile_and_float4_on_both_sides():
    for m, bm in ((32, 32), (33, 64)):
        assert one(recs("conv1x1_fwd", [A16] * 4, [2, 24, m, 64]), "gemm2")["bm"] == bm
    r = one(recs("conv1x1_fwd", [A16] * 4, [2, 24, 48, 64]), "gemm2")
    assert (r["kernel"], r["vec_b"], r["vec_c"], r["grid"]) == ("gemm2_kernel<64>", 1, 1, (1, 1, 2))
    r = one(recs("conv1x1_fwd", [A16 + 4, A16, None, A16], [2, 24, 48, 64]), "gemm2")       # x: B of the forward
    assert (r["vec_b"], r["vec_c"]) == (0, 1)
    r = one(recs("conv1x1_fwd", [A16, A16, None, A16 + 4], [2, 24, 48, 64]), "gemm2")
    assert (r["vec_b"], r["vec_c"]) == (1, 0)
    r = one(recs("conv1x1_fwd", [A16] * 4, [2, 24, 48, 63]), "gemm2")                       # HW % 4
    assert (r["vec_b"], r["vec_c"]) == (0, 0)
    r = one(recs("conv1x1_bwd", [A16, A16, A16 + 4, A16, None, None], [2, 24, 48, 64]), "gemm2")   # dgrad: B = dy, C = dx
    assert (r["bm"], r["vec_b"], r["vec_c"]) == (32, 0, 1)


def test_bn_float4_slices_and_apply_grid_on_both_sides():
    fwd = lambda x, y, n, hw: recs("bn_train_fwd", [x, A16, A16, A16, A16, y, A16, A16, A16], [n, 4, hw, 1])
    rs = fwd(A16, A16, 2, 64)
    assert [r["kernel"] for r in rs] == ["memset", "bn_stats_kernel", "bn_finalize_kernel", "bn_apply_kernel"]
    assert rs[0]["bytes"] == 2 * 4 * 8 and rs[2]["block"] == 128
    assert (one(rs, "bn_stats")["vec"], one(rs, "bn_apply")["vec"]) == (1, 1)
    rs = fwd(A16, A16 + 4, 2, 64)
    assert (one(rs, "bn_stats")["vec"], one(rs, "bn_apply")["vec"]) == (1, 0)
    rs = fwd(A16 + 4, A16, 2, 64)
    assert (one(rs, "bn_stats")["vec"], one(rs, "bn_apply")["vec"]) == (0, 0)
    rs = fwd(A16, A16, 2, 63)
    assert (one(rs, "bn_stats")["vec"], one(rs, "bn_apply")["vec"]) == (0, 0)
    for n, hw, slices in ((1, 4096, 1), (3, 4096, 3), (4, 4096, 4), (200, 1600, 64)):
        r = one(fwd(A16, A16, n, hw), "bn_stats")
        assert (r["slices"], r["grid"]) == (slices, (4, slices, 1)), (n, hw)
        bwd = recs("bn_train_bwd", [A16] * 10, [n, 4, hw, 1])
        assert one(bwd, "bn_bwd_reduce")["slices"] == slices
    for hw, gy in ((1024, 1), (1025, 2)):
        assert one(fwd(A16, A16, 2, hw), "bn_apply")["grid"] == (8, gy, 1)
    ev = lambda dx: recs("bn_eval_bwd", [A16] * 6 + [dx, None, None, None], [2, 4, 64, 1])
    assert one(ev(A16), "bn_eval_bwd_apply")["vec"] == 1 and one(ev(A16 + 4), "bn_eval_bwd_apply")["vec"] == 0


def test_wgrad_kernel_and_chunks_on_both_sides():
    def wg(n, k, m, hw, sms=132):
        rs = recs("conv1x1_bwd", [A16, A16, A16, None, A16, None], [n, k, m, hw], sms)
        assert rs[0]["kernel"] == "memset" and rs[0]["bytes"] == 4 * k * m                   # the op passes no scratch: atomics
        r = one(rs, "wgrad")
        return r["kernel"], r["chunks"], r["partial"], r["grid"]
    assert wg(2, 24, 48, 64) == ("wgrad_rows_kernel<24,3>", 1, 0, (2, 2, 1))
    assert wg(2, 24, 72, 1600)[:2] == ("wgrad_rows_kernel<24,3>", 7)
    assert wg(2, 16, 16, 64)[:2] == ("wgrad1x1_kernel<32>", 1)
    assert wg(2, 16, 16, 81)[:2] == ("wgrad1x1_kernel<32>", 2)
    assert wg(2, 72, 80, 16)[:2] == ("wgrad1x1_kernel<64>", 1)
    assert wg(4, 96, 96, 900)[:2] == ("wgrad1x1_kernel<64>", 15)
    assert wg(2, 48, 48, 64)[0] == "wgrad1x1_kernel<64>"                                      # K = 48: the tiled kernel
    assert wg(4, 96, 96, 900, sms=16)[1] < 15                                                  # fewer SMs, fewer slices


def test_wgrad_partial_sums_until_the_scratch_is_full():
    """The trainer offers a 4 M-float scratch for per-block partial sums: at 64 x 352 x 352 every 1x1 weight gradient fits; at
    203 x 32 x 32 fpn.conv1x1_2 (288 -> 72 on 2 x 2 maps: 203 x 72 x 288 floats) does not and takes the memset + atomics."""
    import yfv2_engine

    def fpn2(shape):
        lib, t = trainer(*shape)
        try:
            ops, tens, _ = yfv2_engine.trainer_program(t)
            rs = yfv2_engine.trainer_launches(t, sms=132)
        finally:
            lib.yfv2_trainer_destroy(t)
        i = next(i for i, o in enumerate(ops) if o["kind"] == "pw" and tens[o["a"]]["C"] == 288)
        return [r for r in rs if r["op"] == i and r["bwd"]], [r for r in rs if r["kernel"].startswith("wgrad1x1") or "rows" in r["kernel"]]
    mine, every = fpn2((64, 352, 352, 3, 80))
    assert all(r["partial"] for r in every)
    assert [r["kernel"] for r in mine] == ["gemm2_kernel<64>", "wgrad1x1_kernel<64>", "wgrad_reduce_kernel"]
    mine, _ = fpn2((203, 32, 32, 3, 80))
    assert [r["kernel"] for r in mine] == ["gemm2_kernel<64>", "memset", "wgrad1x1_kernel<64>"] and not mine[2]["partial"]
    assert mine[1]["bytes"] == 72 * 288 * 4


def test_trainer_records_follow_the_program():
    import yfv2_engine
    lib, t = trainer(2, 64, 96, 3, 80)
    try:
        ops, _, _ = yfv2_engine.trainer_program(t)
        rs = yfv2_engine.trainer_launches(t, workspace=256, sms=132)
        assert yfv2_engine.trainer_launches(t, workspace=260, sms=132) != rs                  # the workspace decides float4 access
        nbwd = len(yfv2_engine.trainer_backward_plan(t))
    finally:
        lib.yfv2_trainer_destroy(t)
    fwd = [r for r in rs if not r["bwd"]]
    assert [r["op"] for r in fwd] == sorted(r["op"] for r in fwd) and {r["op"] for r in fwd} == set(range(len(ops)))
    bwd_ops = [r["op"] for r in rs if r["bwd"] and r["op"] >= 0]
    assert bwd_ops == sorted(bwd_ops, reverse=True) and len(set(bwd_ops)) == nbwd
    assert rs[-1]["op"] == -1 and rs[-1]["kernel"] == "axpy_kernel" and rs[-1]["accumulate"] == 0
    assert all(r["grid"][0] <= 16 * 132 for r in rs if r["kernel"] in ("chan_copy_kernel", "axpy_kernel"))


def test_hooks_refuse_what_the_calls_refuse():
    import yfv2_engine
    lib = yfv2_engine.lib()
    fake = ctypes.c_void_p(16)
    cases = [("conv1x1_fwd", [None, A16, None, A16], [2, 24, 48, 64]), ("conv1x1_bwd", [A16] * 6, [0, 24, 48, 64]),
             ("dwconv_fwd", [A16] * 3, [2, 8, 7, 9, 4, 1]), ("stem_fwd", [A16] * 3, [2, 24, 7, 8]),
             ("bn_train_fwd", [A16] * 9, [1, 8, 1, 1]), ("bn_eval_bwd", [A16] * 6 + [None] * 4, [2, 4, 64, 1]),
             ("maxpool_bwd", [A16, None, A16], [2, 3, 3]), ("upsample2_fwd", [None, A16], [2, 3, 3])]
    for name, ptrs, ints in cases:
        args = [ctypes.c_void_p(p) if p is not None else None for p in ptrs] + ints
        rc = getattr(lib, "yfv2_op_" + name)(*args, None)
        msg = lib.yfv2_last_error()
        assert rc < 0, name
        with pytest.raises(yfv2_engine.Yfv2Error) as e:
            recs(name, ptrs, ints)
        assert ("(%d): %s" % (rc, msg.decode())) in str(e.value), (name, str(e.value))
    with pytest.raises(yfv2_engine.Yfv2Error, match="takes 9 pointers and 4 integers, got 9 and 3"):
        recs("bn_train_fwd", [A16] * 9, [2, 4, 64])                       # a short argument list is refused, not read past
    n = ctypes.c_int()
    assert lib.yfv2_op_debug_launches(99, (ctypes.c_void_p * 1)(), (ctypes.c_int * 1)(), 0, None, 0, ctypes.byref(n)) < 0
    lib_, t = trainer(2, 32, 32, 3, 80)
    try:
        yfv2_engine.trainer_set_mode(t, (False,) * 225, None)
        ptrs = (ctypes.c_void_p * 225)(*([16] * 225))
        rc = lib.yfv2_train_backward(t, fake, ptrs, ptrs, ptrs, fake, 0, fake, None)
        msg = lib.yfv2_last_error().decode()
        assert rc < 0 and "no parameter is trainable" in msg
        with pytest.raises(yfv2_engine.Yfv2Error) as e:
            yfv2_engine.trainer_launches(t)
        assert ("(%d): %s" % (rc, msg)) in str(e.value)
    finally:
        lib.yfv2_trainer_destroy(t)
