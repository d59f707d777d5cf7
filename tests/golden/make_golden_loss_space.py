"""Generates tests/golden/loss_space.npz by running the REAL reference build_target / compute_loss (utils/loss.py, imported from
/root/reference, with make_golden.py's shims) on the small cases of tests/loss_space.py.

    python tests/golden/make_golden_loss_space.py [--reference /root/reference]

Per case `<name>_digest` (SHA-256 of the seeded inputs, to catch a changed builder), `<name>_tcls<L>`, `<name>_tbox<L>`,
`<name>_anch<L>`, `<name>_idx<L>` (b, a, gj, gi stacked), `<name>_losses` (lbox, lobj, lcls, loss) and `<name>_grad<i>`
(d(loss)/d(preds[i])).  The large cases (golden=False) are not stored: the tests compare them with the oracle.  The versions go to
tests/golden/META_loss_space.json.
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)


def np_(t):
    return t.detach().cpu().numpy()


def main():
    import loss_space as ls
    from make_golden import install_shims
    ap = argparse.ArgumentParser()
    ap.add_argument("--reference", default="/root/reference")
    args = ap.parse_args()
    install_shims()
    sys.path.insert(0, args.reference)
    import utils.loss as rloss

    dev = torch.device("cpu")
    out = {}
    names = []
    for case in ls.all_cases():
        if not case["golden"]:
            continue
        ls.check_sides(case)
        name, cfg = case["name"], ls.cfg_of(case)
        names.append(name)
        out[name + "_digest"] = ls.input_digest(case)
        preds = [torch.from_numpy(p.copy()).requires_grad_(True) for p in case["preds"]]
        targets = torch.from_numpy(case["targets"].copy())
        tcls, tbox, indices, anch = rloss.build_target(preds, targets.clone(), cfg, dev)
        for L in range(2):
            out["%s_tcls%d" % (name, L)] = np_(tcls[L]); out["%s_tbox%d" % (name, L)] = np_(tbox[L])
            out["%s_anch%d" % (name, L)] = np_(anch[L])
            out["%s_idx%d" % (name, L)] = np.stack([np_(t) for t in indices[L]], 0)
        lb, lo, lc, loss = rloss.compute_loss(preds, targets.clone(), cfg, dev)
        loss.backward()
        out[name + "_losses"] = np.array([lb.item(), lo.item(), lc.item(), loss.item()], np.float64)
        for i, p in enumerate(preds):            # a head the loss never reads (no rows, or one class) has no grad: zeros
            out["%s_grad%d" % (name, i)] = np_(p.grad) if p.grad is not None else np.zeros(p.shape, np.float32)
    np.savez_compressed(os.path.join(HERE, "loss_space.npz"), **out)
    meta = {"torch": torch.__version__, "numpy": np.__version__, "reference_commit": "ac2a5e3",
            "loss_space": "tests/golden/make_golden_loss_space.py: reference utils/loss.py build_target + compute_loss + autograd "
                          "(CPU) on the seeded cases of tests/loss_space.py",
            "cases": names}
    with open(os.path.join(HERE, "META_loss_space.json"), "w") as f:
        json.dump(meta, f)
    print("wrote loss_space.npz: %d cases (torch %s)" % (len(names), torch.__version__))


if __name__ == "__main__":
    main()
