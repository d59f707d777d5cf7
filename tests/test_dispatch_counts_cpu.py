"""CPU: yfv2_debug_set_dispatch and yfv2_engine.simulated_dispatch.  The hook refuses negative settings and restores the previous
one on exit; under it the forward's, the training ops' and the trainer's launch records follow the simulated SM count as the
records for that count do; and the cheap cases of tests/dispatch_counts_traced.py reach every band-walk cell of the forward."""
import ctypes

import pytest

import yfv2  # noqa: F401
import yfv2_engine as eng
import net_dispatch as nd
import dispatch_counts_traced as dc

A16 = 1 << 20                                                       # a 16-byte-aligned address (never dereferenced)


def test_refuses_negative_settings_and_restores_on_exit():
    L = eng.lib()
    assert L.yfv2_debug_set_dispatch(-1, 0) == eng.lib().yfv2_debug_set_dispatch(0, -3) < 0
    assert b"negative" in L.yfv2_last_error()
    with pytest.raises(eng.Yfv2Error, match="negative"):
        with eng.simulated_dispatch(-2):
            pass
    at = lambda: nd.launches(8, 352, 352, sms=0)
    own = at()
    with eng.simulated_dispatch(7):
        seven = at()
        with eng.simulated_dispatch(16, 3):
            assert at() == nd.launches(8, 352, 352, sms=16)
        assert at() == seven
        with pytest.raises(RuntimeError, match="inside"):
            with eng.simulated_dispatch(1):
                raise RuntimeError("inside")
        assert at() == seven
    assert at() == own and seven != own


@pytest.mark.parametrize("sms", dc.SM_COUNTS)
def test_plan_records_follow_the_hook(sms):
    for n, h, w in dc.SHAPES.values():
        for u8 in (False, True):
            with eng.simulated_dispatch(sms):
                got = nd.launches(n, h, w, sms=0, u8=u8)
            assert got == nd.launches(n, h, w, sms=sms, u8=u8), (n, h, w, u8)


def test_persistent_cap_leaves_the_records_alone():
    """the CTA cap changes only the grid a persistent launch runs, not what the records describe"""
    own = nd.launches(8, 352, 352, sms=0)
    with eng.simulated_dispatch(0, 2):
        assert nd.launches(8, 352, 352, sms=0) == own


def pchunk_of(n, k, m, hw, sms):
    return [(r["kernel"], r["pchunk"], r["chunks"], r["partial"], r["grid"]) for r in
            eng.op_launches("conv1x1_bwd", [A16] * 5 + [None], [n, k, m, hw], sms) if r["kernel"].startswith("wgrad")]


def expected_pchunk(rows, units, hw, sms):
    """k_train.cu describe_conv1x1_bwd: halve the slice while the grid has fewer than two (rows) or four (tiled) waves"""
    p = 2048 if rows else 1024
    while p > (256 if rows else 64) and units * ((hw + p - 1) // p) < (2 if rows else 4) * sms:
        p >>= 1
    return p, (hw + p - 1) // p


def test_op_records_follow_the_hook():
    import test_train_ops_space_gpu as sp
    moved = set()
    for n, k, m, h, w, _, _ in sp.PW:
        rows = k == 24 and m % 24 == 0
        bt = 32 if m <= 32 and k <= 32 else 64
        units = n * (m // 24) if rows else -(-m // bt) * -(-k // bt) * n
        for sms in dc.SM_COUNTS:
            with eng.simulated_dispatch(sms):
                got = pchunk_of(n, k, m, h * w, 0)
            assert got == pchunk_of(n, k, m, h * w, sms)
            (_, p, chunks, partial, _), = got
            assert (p, chunks) == expected_pchunk(rows, units, h * w, sms) and not partial      # the op passes no scratch
            moved.add(("pchunk", p != pchunk_of(n, k, m, h * w, 132)[0][1]))
            moved.add(("chunks", chunks != pchunk_of(n, k, m, h * w, 132)[0][2]))
    assert moved >= {("pchunk", True), ("chunks", True)}
    assert [s for c, s in dc.OP_CASES] and all(dc.op_sm_counts(c) for c, _ in dc.OP_CASES)


def trainer(n, h, w, a=3, c=80):
    t = ctypes.c_void_p()
    assert eng.lib().yfv2_trainer_create(ctypes.byref(t), 0, n, h, w, a, c) == 0
    return t


def test_trainer_records_follow_the_hook():
    """the chan_copy / axpy grids (16 x SMs) and the wgrad slices follow the simulated count; at 64 x 352 x 352, 264 SMs slice the
    widest layers so finely that their partial sums no longer fit the trainer's 4 M-float scratch and they take the atomics"""
    for shape, sms, slices_move, to_atomics in (((2, 640, 352), 1, True, False), ((2, 640, 352), 264, False, False),
                                                 ((64, 352, 352), 264, True, True)):
        t = trainer(*shape)
        try:
            with eng.simulated_dispatch(sms):
                got = eng.trainer_launches(t)
            assert got == eng.trainer_launches(t, sms=sms)
            own = eng.trainer_launches(t, sms=132)
        finally:
            eng.lib().yfv2_trainer_destroy(t)
        pick = lambda rs, kinds: [r for r in rs if r["kernel"].startswith(kinds)]         # (a memset precedes an atomic wgrad)
        copies = [(a["grid"], b["grid"]) for a, b in zip(*(pick(rs, ("chan_copy", "axpy")) for rs in (got, own)))]
        assert all(a[0] <= 16 * sms for a, _ in copies) and any(a != b for a, b in copies), (shape, sms)
        wg = list(zip(*(pick(rs, ("wgrad1x1", "wgrad_rows")) for rs in (got, own))))
        assert any(a["chunks"] != b["chunks"] for a, b in wg) == slices_move, (shape, sms)
        for a, b in wg:
            assert a["chunks"] >= b["chunks"] if sms > 132 else a["chunks"] <= b["chunks"]
        assert any(b["partial"] and not a["partial"] for a, b in wg) == to_atomics, (shape, sms)


def test_cheap_cases_reach_every_band_walk_cell():
    """At 132 SMs the walk R > 1 cells need batches of 16 to 128; the simulated counts reach all of them with at most 8 images"""
    walk = {cl for cl in nd.ALL_CELLS if cl[1].startswith("walk")}
    have = set()
    for name, sms in dc.SIM_CASES:
        n, h, w = dc.SHAPES[name]
        assert n <= 8 and max(h, w) <= 1280
        have |= nd.cells(n, h, w, sms=sms)
    assert walk <= have, walk - have
    assert {s for _, s in dc.SIM_CASES} == set(dc.SM_COUNTS)
    assert {name for name, _ in dc.SIM_CASES} == set(dc.SHAPES)


def test_every_simulated_case_changes_a_launch():
    for name, sms in dc.SIM_CASES:
        n, h, w = dc.SHAPES[name]
        assert dc.changed(nd.launches(n, h, w, sms=sms), nd.launches(n, h, w, sms=132)), (name, sms)
