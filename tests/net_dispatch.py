"""Python model of how a forward picks its kernels and cuts images into row bands.

For a plan (N, H, W, A, C) on a GPU with `sms` multiprocessors, `launches()` returns one record per kernel launch of the forward,
in order: the kernel, the fused stages and blocks it covers, the band geometry of banded block launches and the grid wherever the
host code fixes it.  Every constant and rule below restates the C++ source named beside it; tests/test_net_dispatch_cpu.py pins
the launch groups against the library and tests/test_forward_fp64_gpu.py pins kernel names and grids against a profiler trace.
`find_case()` searches shapes and batches for a plan that reaches a given cell (a launch site in a given variant).

What the trace can and cannot confirm: a stride-2 banded launch takes one CTA per band, so its grid (N * bands) pins R through
the band count.  A stride-1 banded launch with more items than SMs runs an occupancy-sized persistent grid, which does not
reveal R; there (e.g. 128 x 640^2: stage2.1-3 at R = 11, stage3.1-7 at R = 8) R, the band count and the partial flag rest
on blk_rows() below restating k_net.cu blk_rows line for line, and a change to either must be made in both."""
import functools
from dataclasses import dataclass

K_THREADS = 256                      # k_net.cu kThreads
K_WARPS = K_THREADS // 32            # k_net.cu kWarps: one 16-pixel tile per warp at a time
K_MAX_CHAIN = 7                      # k_net.cu kMaxChain; plan.cu groups at most 7 stages (i - group < 7)
K_CHAIN_BUDGET = 110 * 1024          # k_net.cu kChainBudget
K_BAND_BUDGET = 110 * 1024           # k_net.cu kBandBudget
K_SMEM_CAP = 227 * 1024              # common.cuh kSmemCap
K_S2_CHUNK = 32                      # k_net.cu kS2Chunk
K_HEAD_TILE = 96                     # k_net.cu / plan.cu kHeadTile
ST_THREADS = 256                     # k_stem.cu ST_THREADS
K_STEM_W = 27 * 24 + 24              # k_stem.cu kStemW
STEM_SMEM_BUDGET = 112 * 1024        # k_stem.cu launch_stem: ~half an SM's shared memory

STAGE_REPEATS = (4, 8, 4)            # plan.cu kStageRepeats
STAGE_WIDTH = (24, 48, 96)           # plan.cu kStageWidth: branch width K of stages 2, 3, 4


def w_stride(n):                     # tc.cuh w_stride
    return n + 8 if n % 16 == 0 else n


def pw_smem_floats(k, np_):          # k_net.cu pw_smem_floats
    return k * w_stride(np_) + 2 * np_


def blk_rin(stride, r):              # k_net.cu blk_rin
    return stride * (r - 1) + 3


def blk_smem_bytes(k, stride, r, wi):            # k_net.cu blk_smem_bytes
    return (2 * pw_smem_floats(k, k) + 12 * k + k * blk_rin(stride, r) * (wi + 2)) * 4


def blk_s2_image_smem_bytes(k, ho, wi):          # k_net.cu blk_s2_image_smem_bytes
    return (3 * pw_smem_floats(k, k) + 24 * k + K_S2_CHUNK * (2 * ho + 1) * (wi + 2)) * 4


def blk_s2_whole_image(k, ho, wo, wi):           # k_net.cu blk_s2_whole_image
    return k == 96 and ho * wo <= 16 * K_WARPS and blk_s2_image_smem_bytes(k, ho, wi) <= K_SMEM_CAP


def blk_s1_chainable(k, h, w):                   # k_net.cu blk_s1_chainable
    b = blk_smem_bytes(k, 1, h, w)
    return b <= K_CHAIN_BUDGET or (k == 96 and b <= K_SMEM_CAP)


@functools.lru_cache(maxsize=None)
def blk_rows(k, stride, ho, wi, n, sms):         # k_net.cu blk_rows
    r = ho
    while r > 1 and blk_smem_bytes(k, stride, r, wi) > K_BAND_BUDGET:
        r -= 1
    while r > 1 and n * -(-ho // r) < 2 * sms:
        r = (r + 1) // 2
    return r


def stem_smem_bytes(tro, two, s):                # k_stem.cu stem_smem_bytes
    cr, ir, wst = 2 * tro + 1, 4 * tro + 3, 4 * two + 12
    return (K_STEM_W + 256 + 3 * ir * wst + 24 * cr * 2 * s + 4) * 4


def stem_tiling(n, h, w, sms):                   # k_stem.cu launch_stem
    ho, wo = h // 4, w // 4
    tiles_x = -(-wo // 44)
    two = -(-wo // tiles_x)
    s = (2 * two + 1 + 3) // 4
    tro = min((ST_THREADS // s - 1) // 2, ho)
    while tro > 1 and stem_smem_bytes(tro, two, s) > STEM_SMEM_BUDGET:
        tro -= 1
    tro = max(tro, 1)
    tiles_y = -(-ho // tro)
    items = n * tiles_x * tiles_y
    return dict(TRo=tro, TWo=two, S=s, tilesX=tiles_x, tilesY=tiles_y, items=items, grid=min(items, 2 * sms))


# ---- the fused stages of a plan (plan.cu yfv2_plan_create) ----------------------------------------------------------------
def blocks():
    """(stage name, K, stride, output resolution index) of the 16 backbone blocks; resolution r is stride 4 * 2**r."""
    out = []
    for st, rep in enumerate(STAGE_REPEATS):
        for j in range(rep):
            out.append(("stage%d.%d" % (st + 2, j), STAGE_WIDTH[st], 2 if j == 0 else 1, st + 1))
    return out


BLOCKS = blocks()
STAGE_NAMES = (["stem"] + [b[0] for b in BLOCKS] + ["fpn.S3", "fpn.S2", "heads2.a", "heads2.b", "heads3.a", "heads3.b"])


def res_hw(h, w, r):
    return h >> (r + 2), w >> (r + 2)


def stage_groups(h, w):
    """plan.cu: the first stage of the launch each stage belongs to."""
    groups = []
    for i in range(len(STAGE_NAMES)):
        g = i
        b, pb = i - 1, i - 2
        if 0 <= pb and b < 16 and BLOCKS[b][2] == 1 and BLOCKS[pb][2] == 1 and BLOCKS[b][1] == BLOCKS[pb][1] \
                and i - groups[i - 1] < K_MAX_CHAIN and blk_s1_chainable(BLOCKS[b][1], *res_hw(h, w, BLOCKS[b][3])):
            g = groups[i - 1]
        groups.append(g)
    return groups


@dataclass(frozen=True)
class Launch:
    first: int                 # fused stages [first, last) of plan.stage_names
    last: int
    kernel: str                # kernel name as demangled, without spaces: "blk_kernel<96,1>", "stem_kernel<true>", ...
    site: str                  # "stem", "stage2.0", "stage2.s1", ..., "fpn.S3", "fpn.S2", "heads2.a", ..., "heads3.b"
    variant: str               # see cell()
    blocks: tuple = ()         # backbone block indices (0-15) the launch runs, in order
    R: int = 0                 # banded block launches: rows per band, number of bands, last band shorter than R
    bands: int = 0
    partial: bool = False
    items: int = 0             # work items the grid walks
    grid: tuple = None         # (x, y, z) where the host code fixes it; None for occupancy-sized persistent grids

    @property
    def names(self):
        return STAGE_NAMES[self.first:self.last]

    @property
    def cell(self):
        return (self.site, self.variant)


def _banded_variant(r, partial):
    return "R=1" if r == 1 else "R>1 partial" if partial else "R>1"


def launches(n, h, w, a=3, c=80, sms=132, u8=False):
    """The kernel launches of one forward of plan (n, h, w, a, c), in order."""
    groups = stage_groups(h, w)
    out = []
    st = stem_tiling(n, h, w, sms)
    out.append(Launch(0, 1, "stem_kernel<%s>" % ("true" if u8 else "false"), "stem", "u8" if u8 else "f32",
                      items=st["items"], grid=(st["grid"], 1, 1)))
    i = 1
    while i <= 16:
        j = i
        while j + 1 <= 16 and groups[j + 1] == groups[i]:
            j += 1
        bl = tuple(range(i - 1, j))
        name, k, stride, res = BLOCKS[i - 1]
        stage = name.split(".")[0]
        ho, wo = res_hw(h, w, res)
        if stride == 2:
            hi, wi = res_hw(h, w, res - 1)
            site = name
            if blk_s2_whole_image(k, ho, wo, wi):
                out.append(Launch(i, j + 1, "blk_s2_image_kernel<96>", site, "s2img", bl, ho, 1, False, n,
                                  (n, 1, 1) if n <= sms else None))
            else:
                r = blk_rows(k, 2, ho, wi, n, sms)
                if blk_smem_bytes(k, 2, r, wi) > K_SMEM_CAP:
                    raise ValueError("block %s: a %d-row band of %d columns does not fit in shared memory" % (name, r, wi))
                bands = -(-ho // r)
                out.append(Launch(i, j + 1, "blk_kernel<%d,2>" % k, site, _banded_variant(r, ho % r != 0), bl, r, bands,
                                  ho % r != 0, n * bands, (n * bands, 1, 1)))       # one CTA per item
        else:
            site = stage + ".s1"
            if len(bl) > 1:
                if blk_smem_bytes(k, 1, ho, wo) > K_CHAIN_BUDGET:
                    out.append(Launch(i, j + 1, "blk_chain_kernel<96>", site, "chain96", bl, ho, 1, False, n,
                                      (n, 1, 1) if n <= sms else None))
                else:
                    out.append(Launch(i, j + 1, "blk_kernel<%d,1>" % k, site, "chain", bl, ho, 1, False, n, (n, 1, 1)))
            else:
                r = blk_rows(k, 1, ho, wo, n, sms)
                bands = -(-ho // r)
                items = n * bands
                out.append(Launch(i, j + 1, "blk_kernel<%d,1>" % k, site, _banded_variant(r, ho % r != 0), bl, r, bands,
                                  ho % r != 0, items, (items, 1, 1) if items <= sms else None))
        i = j + 1
    for idx, name, kin, res in ((17, "fpn.S3", 192, 3), (18, "fpn.S2", 288, 2)):
        hh, ww = res_hw(h, w, res)
        items = n * -(-hh * ww // (16 * K_WARPS))
        out.append(Launch(idx, idx + 1, "fpn_kernel<%d>" % kin, name, "fpn_kernel<%d>" % kin, items=items,
                          grid=(min(items, 2 * sms), 1, 1)))
    for lv in (0, 1):
        hh, ww = res_hw(h, w, 2 + lv)
        items = n * -(-hh * ww // (16 * K_WARPS))
        grid = (min(items, sms), 2, 1)                    # y: cls branch, reg branch
        idx = 19 + 2 * lv
        out.append(Launch(idx, idx + 1, "head_kernel<0>", "heads.a", "head_kernel<0>", items=items, grid=grid))
        if a + c > 2 * K_HEAD_TILE or 4 * a > K_HEAD_TILE:
            raise ValueError("heads: anchors+classes = %d exceeds two %d-column output tiles" % (a + c, K_HEAD_TILE))
        kern = "head_kernel<1>" if a + c <= K_HEAD_TILE else "head2_kernel"
        out.append(Launch(idx + 1, idx + 2, kern, "heads.b", kern, items=items, grid=grid))
    return out


# ---- cells and the search for shapes that reach them ----------------------------------------------------------------------
def cells(n, h, w, a=3, c=80, sms=132, both_inputs=True):
    """The (site, variant) cells a forward of this plan reaches; with both_inputs, the stem with uint8 and with fp32 input."""
    out = {L.cell for L in launches(n, h, w, a, c, sms)}
    if both_inputs:
        out.add(("stem", "u8"))
    return out


SEARCH_SIDES = tuple(range(32, 1024 + 1, 32))
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


# Every cell a launch site could be in.  Cells no plan of the search space reaches are named by unreachable().
ALL_CELLS = frozenset(
    [("stem", "f32"), ("stem", "u8")]
    + [(s, v) for s in ("stage2.0", "stage3.0") for v in ("R=1", "R>1", "R>1 partial")]
    + [("stage4.0", v) for v in ("s2img", "R=1", "R>1", "R>1 partial")]
    + [(s, v) for s in ("stage2.s1", "stage3.s1") for v in ("chain", "R=1", "R>1", "R>1 partial")]
    + [("stage4.s1", v) for v in ("chain", "chain96", "R=1", "R>1", "R>1 partial")]
    + [("fpn.S3", "fpn_kernel<192>"), ("fpn.S2", "fpn_kernel<288>"), ("heads.a", "head_kernel<0>"),
       ("heads.b", "head_kernel<1>"), ("heads.b", "head2_kernel")])


def unreachable(sms=132, **space):
    return sorted(ALL_CELLS - set(reachable(sms, **space)))
