"""CPU checks of two pieces of host-verifiable reasoning behind device code (no GPU, no CUDA library calls).

1. The heads' second half: pw2 -> BN -> shared output conv are consecutive affine maps, which plan.cu's
   fold_head_kernel composes in fp64 into one [M x 72] matrix + bias.  Here the same composition is done with numpy on
   the oracle's tensors and pushed through the oracle: the folded head must reproduce the reference ordering
   (fpn.py DWConvblock tail + detector.py:17-19,35-41) to fp32 round-off.
2. The NMS sort: nms.cuh's bitonic_sort_desc_reg keeps NT*E keys in registers and mixes in-thread compare-exchanges,
   warp shuffles and a few shared-memory steps.  A numpy model of exactly those index / direction rules must sort, and
   every shuffle partner must sit in the same warp.
"""
import numpy as np
import torch
import torch.nn.functional as F

import synth
from oracle import net as onet

BN_EPS = 1e-5


def _fold(sd, head, outs):
    """F = Wout . diag(sc) . Wpw, f = Wout . sh + bias (fp64 accumulate, one rounding to fp32), as fold_head_kernel."""
    p = "fpn.%s.block." % head
    wpw = sd[p + "8.weight"].double().reshape(72, 72)
    g, b = sd[p + "9.weight"], sd[p + "9.bias"]
    m, v = sd[p + "9.running_mean"], sd[p + "9.running_var"]
    invstd = (1.0 / torch.sqrt(v + BN_EPS)).float()
    sc = (invstd * g).float()
    sh = (b - (m * sc).float()).float()
    Ws, bs = [], []
    for name in outs:
        wo = sd[name + ".weight"].double().reshape(-1, 72)
        Ws.append((wo * sc.double()[None, :]) @ wpw)
        bs.append(wo @ sh.double() + sd[name + ".bias"].double())
    return torch.cat(Ws).float(), torch.cat(bs).float()


def test_folded_head_matches_reference_order():
    sd = synth.make_state_dict(3, 80, 3)
    x = synth.make_images(5, 2, 64, 64)
    taps = {}
    with torch.no_grad():
        ref = onet.forward(sd, x, taps=taps)
    for lvl, (S, reg_i) in enumerate((("S2", 0), ("S3", 3))):
        for head, outs, want in (("cls_head_%d" % (lvl + 2), ("output_obj_layers", "output_cls_layers"),
                                  torch.cat((ref[reg_i + 1], ref[reg_i + 2]), 1)),
                                 ("reg_head_%d" % (lvl + 2), ("output_reg_layers",), ref[reg_i])):
            p = "fpn.%s.block." % head
            with torch.no_grad():
                t = F.relu(onet._bn(sd, onet._dw(sd, taps[S], p + "0", 1, 2), p + "1", False, False))
                t = onet._bn(sd, onet._pw(sd, t, p + "3"), p + "4", False, False)
                u = F.relu(onet._bn(sd, onet._dw(sd, t, p + "5", 1, 2), p + "6", False, False))
                Fw, Fb = _fold(sd, head, outs)
                got = F.conv2d(u, Fw.reshape(-1, 72, 1, 1), Fb)
            scale = float(want.abs().max())
            assert float((got - want).abs().max()) <= 2e-5 * max(scale, 1.0), (head, float((got - want).abs().max()), scale)


NT = 256


def _sort_reg_model(keys, E):
    n2 = NT * E
    t = np.arange(NT)
    v = keys.reshape(NT, E).copy()                 # v[t][m] = keys[E t + m]
    k = 2
    smem_steps = 0
    while k <= n2:
        j = k >> 1
        while j > 0:
            if j >= E:
                pt = t ^ (j // E)
                if j >= 32 * E:
                    smem_steps += 1                # partner thread in another warp: shared memory + barriers
                else:
                    assert np.all((pt // 32) == (t // 32))     # __shfl_xor partner is in the same warp
                o = v[pt, :]
                for m in range(E):
                    i = E * t + m
                    keep_max = ((i & k) == 0) == ((i & j) == 0)
                    a, b = v[:, m].copy(), o[:, m]
                    v[:, m] = np.where(keep_max, np.maximum(a, b), np.minimum(a, b))
            else:
                for m in range(E):
                    if (m & j) == 0:
                        i = E * t + m
                        a, b = v[:, m].copy(), v[:, m | j].copy()
                        sw = np.where((i & k) == 0, a < b, a > b)
                        v[:, m] = np.where(sw, b, a)
                        v[:, m | j] = np.where(sw, a, b)
            j >>= 1
        k <<= 1
    return v.reshape(-1), smem_steps


def test_register_bitonic_network_sorts_descending():
    rng = np.random.default_rng(7)
    for E, want_smem in ((1, 6), (2, 6), (4, 6), (8, 6)):
        n2 = NT * E
        for _ in range(3):
            cnt = int(rng.integers(n2 // 2 + 1, n2 + 1))
            keys = np.zeros(n2, dtype=np.uint64)                       # padding zeros, as sort_and_suppress writes them
            hi = rng.permutation(1 << 20)[:cnt].astype(np.uint64) + np.uint64(1)
            keys[:cnt] = hi * np.uint64(1 << 20) + rng.integers(0, 1 << 20, size=cnt).astype(np.uint64)
            out, smem_steps = _sort_reg_model(keys, E)
            assert np.array_equal(out, np.sort(keys)[::-1])
            assert smem_steps == want_smem                              # log2(NT/32) * (log2(NT/32) + 1) / 2 = 6 of the steps


def test_bench_numa_binding_is_harmless_without_a_gpu():
    """bench.bind_to_gpu_node probes pinned H2D bandwidth per NUMA node; without a usable GPU it must leave the affinity alone."""
    import os
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    sys.path.insert(0, root)
    import bench
    before = os.sched_getaffinity(0)
    desc, prev = bench.bind_to_gpu_node(0)
    import torch
    if not torch.cuda.is_available():
        assert desc is None and prev is None
    assert os.sched_getaffinity(0) == before or desc is not None
    if prev:
        os.sched_setaffinity(0, prev)
