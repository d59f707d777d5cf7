"""Regenerates tests/golden/anchors_cases.npz + META_anchors.json from the REAL reference genanchors.py (its kmeans, IOU, avg_IOU,
write_anchors_to_file and main).

    python tests/golden/make_golden_anchors.py [--reference /path/to/Yolo-FastestV2]

genanchors.py uses np.float, which numpy 2 removed: np.float = float is set before the import.  The module's print is wrapped to
bound the iterations: kmeans mutates the centroid array it is given in place and prints `iter t:` after each assignment step,
so the array at the t-th line is the state iteration t used.  The wrapper snapshots it at every line and stops the run
  - at the line after a cluster lost its members (the centroid array holds 0/0 = NaN): EMPTY_CLUSTER at the previous line;
  - at line m + 1 when the case pins m iterations: NOT_CONVERGED at line m;
otherwise kmeans returns by itself: CONVERGED at the last line.  The assignments of the recorded iteration are the reference's
np.argmin of 1 - IOU over that state.  Per case and k the npz holds the initial picks, centroids, assignments, iterations, status,
avg_IOU and the bytes write_anchors_to_file writes for the recorded centroids; per label tree the boxes main() reads, and for
each seed of anchor_cases.TREE_SEEDS the anchors6.txt and anchors1..10.txt main() writes after random.seed(seed)."""
import argparse
import contextlib
import importlib.util
import io
import json
import os
import random
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import anchor_cases as ac  # noqa: E402

ACTIVE, CONVERGED, EMPTY_CLUSTER, NOT_CONVERGED = 0, 1, 2, 3


class Stop(Exception):
    pass


def load_reference(path):
    np.float = float
    spec = importlib.util.spec_from_file_location("ref_genanchors", os.path.join(path, "genanchors.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def run_kmeans(ref, X, C0, m, tmp):
    """(centroids, assignments, iterations, status, anchors file bytes) of one reference kmeans run."""
    C = np.array(C0, dtype=np.float64)
    state = {"t": 0, "snap": None, "status": None}

    def hook(*args, **kw):
        s = " ".join(str(a) for a in args)
        if not s.startswith("iter "):
            return
        if m is not None and state["t"] == m:
            state["status"] = NOT_CONVERGED
            raise Stop
        if state["t"] and np.isnan(C).any():
            state["status"] = EMPTY_CLUSTER
            raise Stop
        state["t"] += 1
        state["snap"] = C.copy()

    ref.print = hook
    path = os.path.join(tmp, "anchors.txt")
    try:
        ref.kmeans(X, C, 0.005, path, ac.INPUT_W, ac.INPUT_H)
        status, cent = CONVERGED, C.copy()
        assert np.array_equal(cent, state["snap"])
    except Stop:
        status, cent = state["status"], state["snap"]
    finally:
        del ref.print
    with np.errstate(all="ignore"):
        a = np.argmin(np.array([1 - ref.IOU(X[i], cent) for i in range(X.shape[0])]), axis=1)
        avg = ref.avg_IOU(X, cent)
        with contextlib.redirect_stdout(io.StringIO()):
            ref.write_anchors_to_file(cent, X, path, ac.INPUT_W, ac.INPUT_H)
    return cent, a.astype(np.int32), state["t"], status, float(avg), open(path, "rb").read()


def run_main(ref, argv, seed):
    """Runs the reference's main(); returns (boxes it read, {file name: bytes}) or raises what it raised.  A run that does not end
    (empty cluster) raises Stop."""
    out = tempfile.mkdtemp()
    got = {}
    kmeans = ref.kmeans

    def capture(X, centroids, *a):
        got["X"] = X.copy()
        C = centroids

        def hook(*args, **kw):
            if " ".join(str(v) for v in args).startswith("iter ") and np.isnan(C).any():
                raise Stop
        ref.print = hook
        try:
            kmeans(X, centroids, *a)
        finally:
            del ref.print

    ref.kmeans = capture
    sys.argv = ["genanchors.py"] + argv + ["--output_dir", out]
    random.seed(seed)
    try:
        with contextlib.redirect_stdout(io.StringIO()):
            ref.main(sys.argv)
    finally:
        ref.kmeans = kmeans
    return got.get("X"), {f: open(os.path.join(out, f), "rb").read() for f in sorted(os.listdir(out))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reference", default="/root/reference")
    args = ap.parse_args()
    ref = load_reference(args.reference)
    arrays, meta = {}, {"cases": {}, "trees": {}}
    tmp = tempfile.mkdtemp()
    for case in ac.CASES:
        name, boxes, ks, _, m = case
        X = boxes()
        arrays[name + "__X"] = X
        meta["cases"][name] = []
        for k, idx in ac.picks(case, X.shape[0]):
            C, a, t, st, avg, txt = run_kmeans(ref, X, X[idx], m, tmp)
            key = "%s__k%d" % (name, k)
            arrays[key + "__init"] = np.array(idx, dtype=np.int64)
            arrays[key + "__C"] = C
            arrays[key + "__a"] = a
            arrays[key + "__iters"] = np.array(t, dtype=np.int32)
            arrays[key + "__status"] = np.array(st, dtype=np.int32)
            arrays[key + "__avg"] = np.array(avg)
            arrays[key + "__txt"] = np.frombuffer(txt, np.uint8)
            meta["cases"][name].append({"k": k, "iterations": t, "status": st, "avg_iou": avg})
            print(name, k, t, st, avg)
    for variant in ac.GOOD_TREES + ac.BAD_TREES:
        root = tempfile.mkdtemp()
        lst = ac.write_tree(root, variant)
        if variant in ac.BAD_TREES:
            try:
                run_main(ref, ["--traintxt", lst], 0)
            except Exception as e:      # noqa: BLE001  (recorded: what the reference raises)
                meta["trees"][variant] = {"raises": type(e).__name__, "message": str(e)}
                continue
            raise AssertionError("the reference read the bad tree %s" % variant)
        meta["trees"][variant] = {"seeds": {}}
        for seed in ac.TREE_SEEDS:
            for nc in (6, 0):
                try:
                    X, files = run_main(ref, ["--traintxt", lst, "--num_clusters", str(nc)], seed)
                except Stop:
                    meta["trees"][variant]["seeds"].setdefault(str(seed), {})[str(nc)] = "does not end"
                    continue
                arrays["tree_%s__dims" % variant] = X
                for f, b in files.items():
                    arrays["tree_%s__s%d__n%d__%s" % (variant, seed, nc, f)] = np.frombuffer(b, np.uint8)
                meta["trees"][variant]["seeds"].setdefault(str(seed), {})[str(nc)] = sorted(files)
        print(variant, meta["trees"][variant])
    np.savez_compressed(os.path.join(HERE, "anchors_cases.npz"), **arrays)
    meta["numpy"] = np.__version__
    with open(os.path.join(HERE, "META_anchors.json"), "w") as f:
        json.dump(meta, f, indent=1, sort_keys=True)
        f.write("\n")


if __name__ == "__main__":
    main()
