"""The kernel launches of a forward as the library chooses them, and the (launch site, variant) cells they fall in.

`launches()` reads the records the forward itself launches from (yfv2_plan_debug_launches: kernel, fused stages, band geometry,
grid, shared memory, heads' window stride) for a host-side plan, so no dispatch rule is restated here.  `cell` maps a record to
its launch site and variant, and `find_case()` searches shapes and batches for a plan that reaches a given cell.  Plans are host
objects, so none of this needs a GPU; tests/test_forward_fp64_gpu.py checks kernel names and grids against a profiler trace."""
import ctypes
import functools
from dataclasses import dataclass

import yfv2  # noqa: F401
import yfv2_engine


@dataclass(frozen=True)
class Launch:
    first: int                 # fused stages [first, last) of stage_names
    last: int
    kernel: str                # kernel name as demangled, without spaces: "walk::blk_kernel<24,2>", "stem_kernel<true>", ...
    names: tuple               # the plan's stage names of [first, last)
    site: str                  # "stem", "stage2.0", "stage2.s1", ..., "fpn.S3", "fpn.S2", "heads.a", "heads.b"
    variant: str               # see _variant()
    R: int = 0                 # block launches: rows per band, number of bands, last band shorter than R
    bands: int = 0
    partial: bool = False
    items: int = 0             # work items the grid walks
    grid: tuple = None         # (x, y, z) where the launch fixes it; None for occupancy-sized persistent grids
    window_stride: int = 0     # heads: channel stride of a staged window slot; 0: the stencils read the planes

    @property
    def blocks(self):
        """backbone block indices (0-15) the launch runs, in order (stage i + 1 is block i)"""
        return tuple(range(self.first - 1, self.last - 1)) if self.site.startswith("stage") else ()

    @property
    def cell(self):
        return (self.site, self.variant)


def block_stride(name):
    """stride of backbone block `name` ("stage3.0" -> 2, "stage3.4" -> 1): the first block of each stage halves the map"""
    return 2 if name.endswith(".0") else 1


def _site(name):
    if name.startswith("stage") and not name.endswith(".0"):
        return name.split(".")[0] + ".s1"
    return "heads" + name[-2:] if name.startswith("heads") else name


def _variant(site, kernel, nblk, R, partial, window_stride):
    if site == "stem":
        return "u8" if kernel == "stem_kernel<true>" else "f32"
    if site.startswith("fpn"):
        return kernel
    if site.startswith("heads"):
        return kernel + (" staged" if window_stride else "")
    if kernel.startswith("blk_chain_kernel"):
        return "chain96"
    if kernel.startswith("blk_s2_image_kernel"):
        return "s2img"
    if nblk > 1:
        return "chain"
    banded = "R=1" if R == 1 else "R>1 partial" if partial else "R>1"
    return "walk " + banded if kernel.startswith("walk::") else banded


def host_plan(n, h, w, fn, a=3, c=80):
    """fn(handle) for a host-side plan (n, h, w, a, c)"""
    L = yfv2_engine.lib()
    p = ctypes.c_void_p()
    yfv2_engine._check(L.yfv2_plan_create(ctypes.byref(p), 0, n, h, w, a, c, 0), "plan_create")
    try:
        return fn(p)
    finally:
        L.yfv2_plan_destroy(p)


def _stage_names(handle):
    L, names = yfv2_engine.lib(), []
    while L.yfv2_plan_stage_name(handle, len(names)) is not None:
        names.append(L.yfv2_plan_stage_name(handle, len(names)).decode())
    return names


STAGE_NAMES = host_plan(1, 64, 64, _stage_names)      # the same for every plan


def _cell(kernel, first, last, R, bands, window_stride, h):
    """(site, variant, partial) of a record of a plan of input height h"""
    site = _site(STAGE_NAMES[first])
    partial = bands != 0 and R * bands != h >> (int(site[5]) + 1)      # stage k runs at stride 2^(k + 1)
    return site, _variant(site, kernel, last - first, R, partial, window_stride), partial


def _launch(d, h):
    site, variant, partial = _cell(d["kernel"], d["first"], d["last"], d["R"], d["bands"], d["window_stride"], h)
    return Launch(d["first"], d["last"], d["kernel"], tuple(STAGE_NAMES[d["first"]:d["last"]]), site, variant, d["R"], d["bands"],
                  partial, d["items"], None if d["persistent"] else d["grid"], d["window_stride"])


def launches(n, h, w, a=3, c=80, sms=132, u8=False):
    """The kernel launches of one forward of plan (n, h, w, a, c) on sms SMs, in order."""
    return host_plan(n, h, w, lambda p: [_launch(d, h) for d in yfv2_engine.plan_launches(p, None, u8, sms)], a, c)


def plan_launches(plan, u8=False, sms=0):
    """The kernel launches of a forward of a yfv2_engine.Plan on its workspace (sms 0: this device's SM count)."""
    return [_launch(d, plan.H) for d in plan.launches(u8, sms)]


# ---- cells and the search for shapes that reach them ----------------------------------------------------------------------
def _raw(handle, sms, buf=(yfv2_engine.LaunchRecord * 64)()):
    """the raw records of an fp32-input forward on a 16-byte-aligned workspace (the search reads tens of thousands of plans)"""
    n = ctypes.c_int()
    yfv2_engine._check(yfv2_engine.lib().yfv2_plan_debug_launches(handle, None, 0, sms, buf, len(buf), ctypes.byref(n)),
                       "plan_debug_launches")
    return buf[:n.value]


def cells(n, h, w, a=3, c=80, sms=132, both_inputs=True):
    """The (site, variant) cells a forward of this plan reaches; with both_inputs, the stem with uint8 and with fp32 input."""
    out = host_plan(n, h, w, lambda p: {_cell(r.kernel.decode(), r.first, r.last, r.R, r.bands, r.window_stride, h)[:2]
                                        for r in _raw(p, sms)}, a, c)
    if both_inputs:
        out.add(("stem", "u8"))
    return out


# Up to 1280 columns: past the walks' fit limits (992 columns at stage3.0, 1024 at stage3.s1, 1152 at stage2.0, 1280 at
# stage2.s1 for plan widths), where the banded K = 24 / 48 kernels run.
SEARCH_SIDES = tuple(range(32, 1280 + 1, 32))
SEARCH_BATCHES = (1, 2, 4, 8, 16, 24, 32, 48, 64, 128, 256)
SEARCH_CLASSES = ((3, 80), (3, 150))


@functools.lru_cache(maxsize=None)
def reachable(sms=132, sides=SEARCH_SIDES, batches=SEARCH_BATCHES, heads=SEARCH_CLASSES):
    """cell -> the cheapest (fewest input pixels) (n, h, w, a, c) that reaches it, over the search space."""
    best = {}
    for h in sides:
        for w in sides:
            for n in batches:
                for a, c in heads:
                    cost = n * h * w
                    for cl in cells(n, h, w, a, c, sms):
                        if cl not in best or cost < best[cl][0]:
                            best[cl] = (cost, (n, h, w, a, c))
    return {cl: v[1] for cl, v in best.items()}


def find_case(cell, sms=132, **space):
    """The cheapest plan (n, h, w, a, c) of the search space whose forward reaches `cell`, or None."""
    return reachable(sms, **space).get(cell)


_BANDED = ("R=1", "R>1", "R>1 partial")
_WALK = tuple("walk " + b for b in _BANDED)
# Every cell a launch site could be in within the search space.  Cells no plan of the search space reaches are named by
# unreachable().  Not in it: the banded stride-2 K = 24 / 48 kernels with R > 1 (past the walk's fit limit a band of two rows
# exceeds kBandBudget), stage2.s1 with partial banded bands, and the heads reading their stencils from the planes except head2_kernel
# (maps of one or two columns and 128 rows or more, or 2560 columns and more: tests/test_heads_gpu.py runs those).
ALL_CELLS = frozenset(
    [("stem", "f32"), ("stem", "u8")]
    + [(s, v) for s in ("stage2.0", "stage3.0") for v in ("R=1",) + _WALK]
    + [("stage4.0", v) for v in ("s2img",) + _BANDED]
    + [("stage2.s1", v) for v in ("chain", "R=1", "R>1") + _WALK]
    + [("stage3.s1", v) for v in ("chain",) + _BANDED + _WALK]
    + [("stage4.s1", v) for v in ("chain", "chain96") + _BANDED]
    + [("fpn.S3", "fpn_kernel<192>"), ("fpn.S2", "fpn_kernel<288>"), ("heads.a", "head_kernel<0> staged")]
    + [("heads.b", k) for k in ("head_kernel<1> staged", "head2_kernel", "head2_kernel staged")])


def unreachable(sms=132, **space):
    return sorted(ALL_CELLS - set(reachable(sms, **space)))
