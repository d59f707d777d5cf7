"""The Python model of the forward's launch selection (tests/net_dispatch.py) against the library's host-side plans: the chain
groups and the launch count over a sweep of shapes, including both sides of every selection boundary.  Plans are host objects,
so this needs no GPU; kernel names and grids are checked against a profiler trace in tests/test_forward_fp64_gpu.py."""
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


def host_plan(n, h, w, a=3, c=80):
    import yfv2_engine
    lib = yfv2_engine.lib()
    p = ctypes.c_void_p()
    assert lib.yfv2_plan_create(ctypes.byref(p), 0, n, h, w, a, c, 0) == 0, lib.yfv2_last_error()
    names, k = [], ctypes.c_int()
    while lib.yfv2_plan_stage_name(p, len(names)) is not None:
        names.append(lib.yfv2_plan_stage_name(p, len(names)).decode())
    groups = [lib.yfv2_plan_stage_group(p, i) for i in range(len(names))]
    assert lib.yfv2_plan_forward_launches(p, ctypes.byref(k)) == 0
    lib.yfv2_plan_destroy(p)
    return names, groups, k.value


def test_stage_names():
    names, _, _ = host_plan(1, 64, 64)
    assert names == nd.STAGE_NAMES


def test_groups_and_launch_counts_match_the_library_over_shapes():
    shapes = [(h, w) for h in SIDES for w in SIDES] + BOUNDARY
    kinds = set()
    for h, w in shapes:
        _, groups, n_launch = host_plan(1, h, w)
        assert nd.stage_groups(h, w) == groups, (h, w)
        model = nd.launches(1, h, w)
        assert len(model) == n_launch, (h, w)
        assert [(L.first, L.last) for L in model] == [(g, g + groups.count(g)) for g in sorted(set(groups))], (h, w)
        kinds |= {(L.site, L.kernel) for L in model}
    # the sweep reaches every kernel of every site
    assert {("stage4.s1", "blk_kernel<96,1>"), ("stage4.s1", "blk_chain_kernel<96>"), ("stage4.0", "blk_s2_image_kernel<96>"),
            ("stage4.0", "blk_kernel<96,2>"), ("stage3.s1", "blk_kernel<48,1>"), ("stage2.s1", "blk_kernel<24,1>")} <= kinds


@pytest.mark.parametrize("n", [1, 8, 128, 256])
def test_groups_do_not_depend_on_the_batch(n):
    for h, w in BOUNDARY[:12]:
        _, groups, n_launch = host_plan(n, h, w)
        assert nd.stage_groups(h, w) == groups and len(nd.launches(n, h, w)) == n_launch


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
    assert nd.blk_smem_bytes(96, 1, 5, 7) <= nd.K_CHAIN_BUDGET < nd.blk_smem_bytes(96, 1, 5, 8)
    assert nd.blk_smem_bytes(96, 1, 14, 21) <= nd.K_SMEM_CAP < nd.blk_smem_bytes(96, 1, 15, 21)
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


def test_stride2_grids_are_one_cta_per_band():
    for n, h, w in [(256, 352, 352), (128, 640, 640), (24, 864, 160)]:
        for L in nd.launches(n, h, w):
            if L.kernel.startswith("blk_kernel") and L.kernel.endswith(",2>"):
                assert L.grid == (n * L.bands, 1, 1) and L.bands == -(-nd.res_hw(h, w, nd.BLOCKS[L.blocks[0]][3])[0] // L.R)


def test_every_cell_is_reachable():
    """Every (site, variant) cell, banded blk_kernel<96, 1> with R > 1 included, is reached by some plan of the search space."""
    assert nd.unreachable() == []
    n, h, w, a, c = nd.find_case(("stage4.s1", "R>1"))
    assert ("stage4.s1", "R>1") in nd.cells(n, h, w, a, c)
