#!/usr/bin/env python
"""The reference's genanchors.py on the GPU: IoU k-means over the (w, h) of every box in a training list, written as the
anchors line of a `.data` file.

    python yolo-fastestv2_b200/genanchors.py --traintxt data/train.txt --output_dir ./ --seed 0

It takes the reference's arguments (--traintxt, --output_dir, --num_clusters, 0 for k = 1..10, --input_width, --input_height) and
writes the same anchors{k}.txt: for a given --seed the bytes the reference writes after random.seed(seed).  The k-means runs on
the device (yfv2_engine.kmeans_anchors), bit-identical to the reference iteration by iteration.  Added:
  --seed S       seeds Python's `random` for the initial picks (without it they are unseeded, as in the reference);
  --restarts R   R runs per k from consecutive picks of the same stream, advanced together; the converged run with the best
                 average IoU is written (R = 1 is the reference's run);
  --max-iter M   a run stops after M iterations (the reference has no limit).
Where the reference never stops (a cluster left without members divides 0 by 0), the run ends as "empty cluster".  One line
per run is printed instead of the reference's per-iteration progress.  Exits with status 1 when some k had no converged run;
its file is not written."""
import argparse
import os
import sys

_PKG = os.path.dirname(os.path.abspath(__file__))
if _PKG not in sys.path:
    sys.path.insert(0, _PKG)

import yfv2_engine                  # noqa: E402
from utils import anchors as ua     # noqa: E402


def main(argv=None):
    p = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    p.add_argument("--traintxt", default="", help="path to traintxt")
    p.add_argument("--output_dir", default="./", type=str, help="Output anchor directory")
    p.add_argument("--num_clusters", default=6, type=int, help="number of clusters (0: 1 through 10)")
    p.add_argument("--input_width", default=352, type=int, help="model input width")
    p.add_argument("--input_height", default=352, type=int, help="model input height")
    p.add_argument("--seed", default=None, type=int, help="seed of the initial picks (default: unseeded)")
    p.add_argument("--restarts", default=1, type=int, help="k-means runs per k; the best converged one is written")
    p.add_argument("--max-iter", dest="max_iter", default=1000, type=int, help="iterations after which a run stops")
    args = p.parse_args(argv)
    if args.restarts < 1 or args.max_iter < 1:
        p.error("--restarts and --max-iter must be at least 1")

    if not os.path.exists(args.output_dir):
        os.mkdir(args.output_dir)
    dims = ua.read_label_dims(args.traintxt)
    rng = ua.seeded_rng(args.seed)
    ks = range(1, 11) if args.num_clusters == 0 else [args.num_clusters]
    failed = []
    for k in ks:
        init = ua.initial_picks(rng, dims.shape[0], k, args.restarts)
        res = yfv2_engine.kmeans_anchors(dims, k, init, args.max_iter)
        status, iters, avg = res.status.cpu().numpy(), res.iterations.cpu().numpy(), res.avg_iou.cpu().numpy()
        for r in range(args.restarts):
            print("k=%d run %d: %s after %d iterations, avg IoU %f" % (k, r, ua.STATUS_NAMES[status[r]], iters[r], avg[r]))
        best = ua.best_run(status, avg)
        if best is None:
            print("k=%d: no run converged; anchors%d.txt not written" % (k, k), file=sys.stderr)
            failed.append(k)
            continue
        path = os.path.join(args.output_dir, "anchors%d.txt" % k)
        with open(path, "w") as f:
            f.write(ua.anchors_text(res.centroids[best].cpu().numpy(), avg[best], args.input_width, args.input_height))
        print("k=%d: run %d -> %s" % (k, best, path))
    return 1 if failed else 0


if __name__ == "__main__":
    sys.exit(main())
