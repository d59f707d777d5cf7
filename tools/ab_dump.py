#!/usr/bin/env python
"""A/B helper: dumps the six head tensors and every block tap for a few seeded inputs to an .npz, so two builds can be
compared bit for bit (e.g. `ab_dump.py old.npz` in a build of the parent commit, `ab_dump.py new.npz` in a build of the
change, then `ab_dump.py --cmp old.npz new.npz`)."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)
import numpy as np  # noqa: E402


def dump(path):
    import torch
    import yfv2  # noqa: F401
    import synth
    import model.detector as det
    out = {}
    for tag, (n, h, w) in {"a": (3, 352, 352), "b": (2, 64, 96), "c": (1, 640, 640), "d": (5, 32, 32)}.items():
        m = det.Detector(80, 3, True)
        m.load_state_dict(synth.make_state_dict(11))
        m = m.cuda().eval()
        x = synth.make_images(12, n, h, w).cuda()
        preds = m(x)
        for i, p in enumerate(preds):
            out["%s_pred%d" % (tag, i)] = p.cpu().numpy()
        plan = next(iter(m._plans.values()))
        names = plan.stage_names
        done = 0
        bi = 0
        for i, nm in enumerate(names):           # one stage at a time: every block output is tapped before it is recycled
            last_of_block = i + 1 == len(names) or names[i + 1].split("/")[0] != nm.split("/")[0]
            if not last_of_block:
                continue
            plan.forward_range(x, preds, done, i + 1)
            done = i + 1
            if nm.startswith(("stem", "stage")):
                out["%s_tap%d" % (tag, bi)] = plan.debug_gather(bi).cpu().numpy()
                bi += 1
    np.savez(path, **out)
    print("wrote", path, len(out), "arrays")


def cmp(a, b):
    A, B = np.load(a), np.load(b)
    bad, close, worst = 0, 0, 0.0
    for k in A.files:
        same = np.array_equal(A[k], B[k])
        if not same:
            d = float(np.abs(A[k] - B[k]).max())
            tol = 1e-5 * max(1.0, float(np.abs(A[k]).max()))
            worst = max(worst, d)
            if d > tol:
                bad += 1
                print("DIFF %-12s max|d| %.3e (tol %.1e)" % (k, d, tol))
            else:
                close += 1
    print("compared %d arrays: %d bit-identical, %d within 1e-5, %d beyond (worst |d| %.3e)"
          % (len(A.files), len(A.files) - close - bad, close, bad, worst))
    return bad


if __name__ == "__main__":
    if sys.argv[1] == "--cmp":
        sys.exit(1 if cmp(sys.argv[2], sys.argv[3]) else 0)
    dump(sys.argv[1])
