"""Generates tests/golden/count_cases.npz with the REAL cv2 (OpenCV 4.13, x86 build): cv2.pointPolygonTest(contour, (x, y), False)
of float32 contours (convex, concave, self-intersecting, with horizontal edges and off-grid vertices) at their vertices, on
their edges and horizontal edges, at float64 points that round onto or off an edge in float32, on a grid and at seeded points;
and of int32 contours against their float32 copies.  OpenCV is present in the build container only, so no test calls cv2: they
compare tests/count_oracle.py against what this script froze.

    python tests/golden/make_golden_count.py

`contours` float32 [C, 64, 2] (padded), `nverts` int32 [C], `poly` int32 [N] (the contour of each point), `points` float64
[N, 2] (what was given to cv2), `result` int8 [N] (cv2's -1 / 0 / 1); `int_contours` int32 [D, 64, 2], `int_nverts` [D],
`int_poly` [M], `int_points` float64 [M, 2], `int_result` int8 [M] (cv2 on the int32 contour, asserted equal to cv2 on its float32
copy).  The script asserts that tests/count_oracle.py gives cv2's answer on every case.  The versions go to
tests/golden/META_count.json.
"""
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))

PMAX = 64


def polygons():
    star = [(100 + 80 * np.cos(a) * (1 if k % 2 == 0 else 0.4), 100 + 80 * np.sin(a) * (1 if k % 2 == 0 else 0.4))
            for k, a in enumerate(np.linspace(0, 2 * np.pi, 10, endpoint=False))]
    pentagram = [(200 + 90 * np.cos(a), 200 + 90 * np.sin(a)) for a in np.linspace(0, 4 * np.pi, 5, endpoint=False) - np.pi / 2]
    return [
        [(100, 20), (300, 20), (300, 200), (100, 200)],                                 # square, horizontal and vertical edges
        [(0, 0), (100, 0), (100, 90), (0, 90)],                                         # its right edge is x = 100
        [(0, 0), (120, 0), (120, 40), (40, 40), (40, 120), (0, 120)],                   # L: concave
        star,                                                                           # concave, off-grid vertices
        [(0, 0), (100, 100), (100, 0), (0, 100)],                                       # bow-tie: self-intersecting
        pentagram,                                                                      # self-intersecting, odd-even inside
        [(10.25, 5.5), (90.75, 5.5), (60.1, 80.3)],                                     # triangle, off-grid
        [(0, 0), (50, 0), (50, 50), (50, 100), (0, 100), (0, 50)],                      # collinear vertices
        [(-1e4, -1e4), (1e4, -1e4), (1e4, 1e4), (-1e4, 1e4)],                           # large
    ]


def points_for(v, rng):
    v = np.asarray(v, np.float64)
    n = len(v)
    pts = [tuple(p) for p in v]                                                         # vertices
    for i in range(n):
        a, b = v[i - 1], v[i]
        for t in (0.5, 0.25, 1 / 3):
            pts.append(tuple(a + t * (b - a)))                                          # on edges (as far as fp allows)
        if a[1] == b[1]:
            pts += [((a[0] + b[0]) / 2, a[1]), (min(a[0], b[0]) - 1, a[1]), (max(a[0], b[0]) + 1, a[1])]
        m = (a + b) / 2
        for d in (1e-6, 1e-5, 1e-3, 0.5):                                               # rounding onto / off the edge in float32
            pts += [(m[0] + d, m[1]), (m[0] - d, m[1]), (m[0], m[1] + d), (m[0], m[1] - d)]
    lo, hi = v.min(0) - 10, v.max(0) + 10
    gx = np.linspace(lo[0], hi[0], 13)
    gy = np.linspace(lo[1], hi[1], 13)
    pts += [(float(np.round(x)), float(np.round(y))) for x in gx for y in gy]
    pts += [tuple(p) for p in rng.uniform(lo, hi, (200, 2))]
    return pts


def main():
    import cv2
    import count_oracle as co
    rng = np.random.default_rng(7)
    polys = polygons()
    contours = np.zeros((len(polys), PMAX, 2), np.float32)
    nverts = np.array([len(p) for p in polys], np.int32)
    poly, points, result = [], [], []
    for c, p in enumerate(polys):
        contours[c, :len(p)] = np.asarray(p, np.float32)
        cf = contours[c, :len(p)]
        for q in points_for(p, rng) + [(100.000001, 45.0), (100.00001, 45.0)]:
            r = cv2.pointPolygonTest(cf, (float(q[0]), float(q[1])), False)
            poly.append(c)
            points.append(q)
            result.append(int(r))
            assert co.point_polygon(cf, np.float32(q[0]), np.float32(q[1])) == int(r), (c, q, r)
    assert cv2.pointPolygonTest(contours[1, :4], (100.000001, 45.0), False) == 0
    assert cv2.pointPolygonTest(contours[1, :4], (100.00001, 45.0), False) == -1

    int_contours = np.zeros((24, PMAX, 2), np.int32)
    int_nverts = np.zeros((24,), np.int32)
    int_poly, int_points, int_result = [], [], []
    for d in range(24):
        n = int(rng.integers(3, 12))
        vi = rng.integers(0, 64, (n, 2)).astype(np.int32)
        int_contours[d, :n], int_nverts[d] = vi, n
        vf = vi.astype(np.float32)
        pts = [(float(x), float(y)) for x in range(-2, 67, 3) for y in range(-2, 67, 3)]      # integer points: cv2's integer branch
        pts += [tuple(p) for p in rng.uniform(-2, 66, (150, 2))] + [tuple(p) for p in vi.astype(np.float64)]
        for q in pts:
            ri = cv2.pointPolygonTest(vi, q, False)
            rf = cv2.pointPolygonTest(vf, q, False)
            assert ri == rf, (d, q, ri, rf)
            assert co.point_polygon(vf, np.float32(q[0]), np.float32(q[1])) == int(ri), (d, q, ri)
            int_poly.append(d)
            int_points.append(q)
            int_result.append(int(ri))

    np.savez_compressed(os.path.join(HERE, "count_cases.npz"), contours=contours, nverts=nverts, poly=np.array(poly, np.int32),
                        points=np.array(points, np.float64), result=np.array(result, np.int8), int_contours=int_contours,
                        int_nverts=int_nverts, int_poly=np.array(int_poly, np.int32), int_points=np.array(int_points, np.float64),
                        int_result=np.array(int_result, np.int8))
    meta = {"opencv": cv2.__version__, "numpy": np.__version__,
            "count_cases": "tests/golden/make_golden_count.py: cv2.pointPolygonTest(contour, (x, y), False) of float32 contours "
                           "(convex, concave, self-intersecting) at vertices, edges, float32 rounding edges, a grid and seeded "
                           "points, and of int32 contours against their float32 copies (x86 build)"}
    with open(os.path.join(HERE, "META_count.json"), "w") as f:
        json.dump(meta, f)
    print(len(points), "float32-contour points,", len(int_points), "int32-contour points;", np.bincount(np.array(result) + 1))


if __name__ == "__main__":
    main()
