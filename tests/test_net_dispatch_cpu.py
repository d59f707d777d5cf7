"""The forward's launch records (yfv2_plan_debug_launches, through tests/net_dispatch.py) against the library's host-side plans:
the launch groups and counts over a sweep of shapes, both sides of every selection boundary, and the band geometries of the
benchmark's batches.  Plans are host objects, so this needs no GPU; kernel names and grids are checked against a profiler trace in
tests/test_forward_fp64_gpu.py."""
import ctypes

import pytest

import yfv2  # noqa: F401
import net_dispatch as nd

SIDES = list(range(32, 1024 + 1, 32))
# both sides of every boundary: stage4.0 on whole images up to Ho*Wo = 128 (512x256, 16x8) and banded at 136 (544x256, 17x8);
# K = 96 chains on blk_kernel up to (h+2)(w+2) = 69 (160x224: 7x9 = 63; 160x256: 7x10 = 70) and on blk_chain_kernel up to 381
# (480x672: 17x23 = 391 is past it; 448x672: 16x23 = 368 within); K = 48 chains up to (h+2)(w+2) = 454 at stride 16
BOUNDARY = [(512, 256), (544, 256), (256, 512), (256, 544), (160, 224), (160, 256), (224, 160), (448, 672), (480, 672),
            (672, 448), (672, 480), (320, 320), (352, 352), (320, 352), (32, 1024), (1024, 32), (4096, 32)]


def groups_and_count(n, h, w):
    import yfv2_engine
    lib = yfv2_engine.lib()

    def read(p):
        k = ctypes.c_int()
        assert lib.yfv2_plan_forward_launches(p, ctypes.byref(k)) == 0
        return [lib.yfv2_plan_stage_group(p, i) for i in range(len(nd.STAGE_NAMES))], k.value
    return nd.host_plan(n, h, w, read)


def test_stage_names():
    assert nd.STAGE_NAMES == (["stem"] + ["stage2.%d" % j for j in range(4)] + ["stage3.%d" % j for j in range(8)]
                              + ["stage4.%d" % j for j in range(4)] + ["fpn.S3", "fpn.S2", "heads2.a", "heads2.b", "heads3.a",
                                                                       "heads3.b"])


def test_groups_and_launch_counts_match_the_library_over_shapes():
    """One record per launch group of yfv2_plan_stage_group, yfv2_plan_forward_launches of them, in stage order."""
    shapes = [(h, w) for h in SIDES for w in SIDES] + BOUNDARY
    kinds = set()
    for h, w in shapes:
        groups, n_launch = groups_and_count(1, h, w)
        ls = nd.launches(1, h, w)
        assert len(ls) == n_launch, (h, w)
        assert [(L.first, L.last) for L in ls] == [(g, g + groups.count(g)) for g in sorted(set(groups))], (h, w)
        kinds |= {(L.site, L.kernel) for L in ls}
    # the sweep reaches every kernel of every site
    assert {("stage4.s1", "blk_kernel<96,1>"), ("stage4.s1", "blk_chain_kernel<96>"), ("stage4.0", "blk_s2_image_kernel<96>"),
            ("stage4.0", "blk_kernel<96,2>"), ("stage3.s1", "blk_kernel<48,1>"), ("stage2.s1", "blk_kernel<24,1>"),
            ("stage3.s1", "walk::blk_kernel<48,1>"), ("stage2.s1", "walk::blk_kernel<24,1>"), ("stage2.0", "walk::blk_kernel<24,2>"),
            ("stage3.0", "walk::blk_kernel<48,2>")} <= kinds


@pytest.mark.parametrize("n", [1, 8, 128, 256])
def test_groups_do_not_depend_on_the_batch(n):
    for h, w in BOUNDARY[:12]:
        groups, n_launch = groups_and_count(n, h, w)
        assert groups == groups_and_count(1, h, w)[0]
        assert [(L.first, L.last) for L in nd.launches(n, h, w)] == [(g, g + groups.count(g)) for g in sorted(set(groups))]
        assert len(nd.launches(n, h, w)) == n_launch


def test_selection_boundaries():
    def kern(n, h, w, site):
        return [L for L in nd.launches(n, h, w) if L.site == site]
    assert kern(8, 512, 256, "stage4.0")[0].kernel == "blk_s2_image_kernel<96>"       # 16 x 8 = 128 output pixels
    assert kern(8, 544, 256, "stage4.0")[0].kernel == "blk_kernel<96,2>"              # 17 x 8 = 136
    assert kern(1, 32, 1024, "stage4.0")[0].variant == "s2img"                        # 1 x 32
    assert [L.kernel for L in kern(1, 160, 224, "stage4.s1")] == ["blk_kernel<96,1>"]         # chain within kChainBudget
    assert [L.kernel for L in kern(1, 160, 256, "stage4.s1")] == ["blk_chain_kernel<96>"]     # past it, within kSmemCap
    assert [L.kernel for L in kern(1, 448, 672, "stage4.s1")] == ["blk_chain_kernel<96>"]
    assert [L.kernel for L in kern(1, 480, 672, "stage4.s1")] == ["blk_kernel<96,1>"] * 3     # past kSmemCap: banded
    # the configs of the benchmark at 132 SMs
    big = {L.site: L for L in nd.launches(256, 352, 352)}
    assert (big["stage2.0"].R, big["stage2.0"].bands, big["stage2.0"].partial) == (5, 9, True)
    assert (big["stage2.s1"].R, big["stage3.0"].R, big["stage3.s1"].R) == (22, 4, 17)
    assert big["stage4.0"].variant == "s2img" and big["stage4.s1"].variant == "chain96"
    big = {L.site: L for L in nd.launches(128, 640, 640)}
    assert (big["stage2.s1"].R, big["stage2.s1"].bands, big["stage2.s1"].partial) == (11, 8, True)
    assert (big["stage3.s1"].R, big["stage4.0"].R, big["stage4.s1"].R) == (8, 1, 1)
    assert [L.kernel for L in nd.launches(2, 96, 128, 3, 150) if L.site == "heads.b"] == ["head2_kernel"] * 2
    assert [L.kernel for L in nd.launches(2, 96, 128, 3, 93) if L.site == "heads.b"] == ["head_kernel<1>"] * 2


def test_walk_fit_limits_at_plan_widths():
    """The band walks fit up to 286 input columns at stage2.0 (K = 24), 122 at stage3.0 (K = 48), 158 at stage2.s1 and 62 at
    stage3.s1: at plan widths (multiples of 32) stage3.0 leaves the walk between 960 and 992 image columns, stage3.s1 between 992
    and 1024, stage2.0 between 1120 and 1152 and stage2.s1 between 1248 and 1280.  No plan reaches the columns in between.  Past
    a limit blk_kernel<K, STRIDE> runs the block, with the same bands and grid."""
    def at(h, w, site):
        return next(L for L in nd.launches(1, h, w) if L.site == site)
    for site, h, walk_w, k in (("stage3.0", 64, 960, "<48,2>"), ("stage3.s1", 128, 992, "<48,1>"), ("stage2.0", 64, 1120, "<24,2>"),
                               ("stage2.s1", 128, 1248, "<24,1>")):
        on, past = at(h, walk_w, site), at(h, walk_w + 32, site)
        assert (on.kernel, past.kernel) == ("walk::blk_kernel" + k, "blk_kernel" + k), site
        assert (on.R, on.bands, on.items, on.grid) == (past.R, past.bands, past.items, past.grid), site
    # at 352^2 the walks keep two CTAs per SM (at most 113 KB each), stepping 4 rows at a time at K = 24 and 3 at K = 48
    import yfv2_engine
    recs = nd.host_plan(256, 352, 352, lambda p: yfv2_engine.plan_launches(p, None, False, 132))
    walks = {r["kernel"]: r for r in recs if r["kernel"].startswith("walk::")}
    assert sorted(walks) == ["walk::blk_kernel<24,1>", "walk::blk_kernel<24,2>", "walk::blk_kernel<48,1>", "walk::blk_kernel<48,2>"]
    assert all(r["smem"] <= 113 * 1024 for r in walks.values())
    assert (walks["walk::blk_kernel<24,1>"]["G"], walks["walk::blk_kernel<48,1>"]["G"]) == (4, 3)


def test_stride2_grids_are_one_cta_per_band():
    for n, h, w in [(256, 352, 352), (128, 640, 640), (24, 864, 160)]:
        for L in nd.launches(n, h, w):
            if L.kernel.endswith(",2>"):
                ho = h >> (int(L.site[5]) + 1)
                assert L.grid == (n * L.bands, 1, 1) and L.bands == -(-ho // L.R), L


def test_bad_arguments_of_the_launch_hook():
    import yfv2_engine
    lib, k = yfv2_engine.lib(), ctypes.c_int()
    assert lib.yfv2_plan_debug_launches(None, None, 0, 0, None, 0, ctypes.byref(k)) < 0
    assert nd.host_plan(1, 64, 64, lambda p: lib.yfv2_plan_debug_launches(p, None, 0, -1, None, 0, ctypes.byref(k))) < 0
    assert nd.host_plan(1, 64, 64, lambda p: lib.yfv2_plan_debug_launches(p, None, 0, 0, None, 1, ctypes.byref(k))) < 0
    assert nd.host_plan(1, 64, 64, lambda p: lib.yfv2_plan_debug_launches(p, None, 0, 0, None, 0, ctypes.byref(k))) == 0
    assert k.value == 13


def test_every_cell_is_reachable():
    """Every (site, variant) cell, banded blk_kernel<96, 1> with R > 1 included, is reached by some plan of the search space."""
    assert nd.unreachable() == []
    n, h, w, a, c = nd.find_case(("stage4.s1", "R>1"))
    assert ("stage4.s1", "R>1") in nd.cells(n, h, w, a, c)
