"""CPU: the training dispatch model (tests/train_dispatch.py) against the native trainer's own program, read through the host-only
hooks yfv2_trainer_debug_ops / _tensors / _layout; the case lists of the fp64 training suites against every cell of the model; and
the refusals that need no device (a BatchNorm over one value per channel)."""
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
        assert layout["gflat_floats"] == sum(pnumel) and layout["wscratch_floats"] == td.K_WSCRATCH_FLOATS
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
    with pytest.raises(ValueError, match="Expected more than 1 value per channel when training"):
        yfv2_engine.check_bn_batch(1, 32, 32)
    with pytest.raises(ValueError):
        yfv2_engine.check_bn_batch(1, 30, 20)                      # the op-by-op path's sizes: stride 32 rounds up to 1 x 1
    for n, h, w in ((2, 32, 32), (1, 32, 64), (1, 64, 32), (1, 66, 64)):
        yfv2_engine.check_bn_batch(n, h, w)
