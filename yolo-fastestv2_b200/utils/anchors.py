"""Host side of the anchor k-means (reference genanchors.py): label parsing, the initial picks, choosing a restart and the
anchors{k}.txt text.  The k-means itself runs on the device (yfv2_engine.kmeans_anchors)."""
import random

import numpy as np

CONVERGED = 1                       # include/yfv2.h YFV2_ANCHOR_CONVERGED
STATUS_NAMES = ("active", "converged", "empty cluster", "not converged")


def label_path(image_path):
    """The label file genanchors.py:135-139 reads for one line of the image list."""
    return image_path.replace("JPEGImages", "labels").replace(".jpg", ".txt").replace(".png", ".txt")


def read_label_dims(traintxt):
    """float64 [N, 2] (w, h) of every box of every label file the list names, in order (genanchors.py:124-147).  Each label line is
    `class x y w h` separated by single spaces; a line that genanchors cannot parse (double space, empty line, a sixth field)
    raises ValueError naming the file and line, and so does a list without any box."""
    with open(traintxt) as f:
        lines = [line.rstrip("\n") for line in f.readlines()]
    dims = []
    for line in lines:
        path = label_path(line)
        with open(path) as f2:
            for n, row in enumerate(f2.readlines(), 1):
                try:
                    w, h = row.rstrip("\n").split(" ")[3:]
                    dims.append((float(w), float(h)))
                except ValueError as e:
                    raise ValueError("%s:%d: %r is not 'class x y w h' separated by single spaces (%s)" % (path, n, row, e)) from None
    if not dims:
        raise ValueError("%s: the label files it lists hold no box" % traintxt)
    return np.array(dims, dtype=np.float64)


def initial_picks(rng, N, k, R=1):
    """int64 [R, k] box indices: run r draws k times rng.randrange(N) right after run r - 1, as genanchors.py:157 draws one run."""
    return np.array([[rng.randrange(N) for _ in range(k)] for _ in range(R)], dtype=np.int64).reshape(R, k)


def best_run(status, avg_iou):
    """Index of the converged run with the largest average IoU (the first on a tie; NaN ranks last), or None when no run
    converged."""
    best = None
    for r, (st, v) in enumerate(zip(status, avg_iou)):
        if st != CONVERGED:
            continue
        if best is None or v > avg_iou[best] or (np.isnan(avg_iou[best]) and not np.isnan(v)):
            best = r
    return best


def anchors_text(centroids, avg_iou, width, height):
    """What write_anchors_to_file (genanchors.py:42-65) writes: the centroids scaled to the input size in float64, in np.argsort
    order of the widths, `w,h` with 2 decimals separated by ", ", then the average IoU with 6 decimals."""
    anchors = np.asarray(centroids, dtype=np.float64) * np.array([float(width), float(height)])
    order = np.argsort(anchors[:, 0])
    return ", ".join("%0.2f,%0.2f" % (anchors[i, 0], anchors[i, 1]) for i in order) + "\n" + "%f\n" % avg_iou


def seeded_rng(seed):
    """genanchors draws from Python's `random`; seed None seeds from the system, as the reference does."""
    return random.Random(seed)
