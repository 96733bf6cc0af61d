#!/usr/bin/env python
"""Measure a mesh against a reference surface on the GPU (sparf_b200.mesh.compare): Chamfer accuracy and completeness,
precision, recall and F-score at a distance threshold, and the Hausdorff distance.

    python tools/compare_mesh.py PRED.ply REF.ply --threshold T [--samples N] [--max-dist D] [--seed S]

Both files are read with mesh.read_ply (ascii or binary little-endian).  A file with faces is sampled with N points
(default 1 000 000) uniformly over its area; a file without a face element is a point cloud (such as DTU's reference
scans) and its points are used as they are.  Distances are exact closest-point distances to the other side's
triangles (or points), capped at D.  Masks and crops are the caller's: filter the points before writing the files.
Prints the metrics, V and F of each side, and the time of each phase (load, sample, grid, query).
"""
import argparse
import math
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
import torch


def build_parser():
    ap = argparse.ArgumentParser()
    ap.add_argument("pred", help="the mesh to score (.ply)")
    ap.add_argument("ref", help="the reference mesh or point cloud (.ply)")
    ap.add_argument("--threshold", type=float, required=True, help="distance threshold of precision, recall, F-score")
    ap.add_argument("--samples", type=int, default=1_000_000, help="surface samples of a side with faces")
    ap.add_argument("--max-dist", type=float, default=float("inf"), help="cap of every distance (default: none)")
    ap.add_argument("--seed", type=int, default=0)
    return ap


def parse_args(ap, argv):
    args = ap.parse_args(argv)
    if not args.threshold > 0:
        ap.error("--threshold must be > 0")
    if args.samples < 0:
        ap.error("--samples must be >= 0")
    if not args.max_dist >= 0:
        ap.error("--max-dist must be >= 0")
    return args


def main(argv=None):
    args = parse_args(build_parser(), argv)
    assert torch.cuda.is_available(), "compare_mesh.py runs on a GPU"
    from sparf_b200 import mesh
    t0 = time.perf_counter()
    sides = []
    for path in (args.pred, args.ref):
        m = mesh.read_ply(path)
        sides.append({k: v.cuda() for k, v in m.items()})
    torch.cuda.synchronize()
    phases = {"load": time.perf_counter() - t0}
    res = mesh.compare(sides[0], sides[1], args.threshold, n_samples=args.samples, max_dist=args.max_dist,
                       seed=args.seed, stats=phases)
    for name, path, m in (("pred", args.pred, sides[0]), ("ref", args.ref, sides[1])):
        faces = m.get("faces")
        print("%s %s: V %d, %s" % (name, path, m["vertices"].shape[0],
                                   "point cloud" if faces is None else "F %d" % faces.shape[0]))
    print("samples: pred %d, ref %d" % (res["n_pred"], res["n_ref"]))
    fmt = lambda x: "nan" if math.isnan(x) else ("inf" if math.isinf(x) else "%.6g" % x)
    print("accuracy %s, completeness %s, chamfer %s" % (fmt(res["accuracy"]), fmt(res["completeness"]),
                                                        fmt(res["chamfer"])))
    print("threshold %g: precision %s, recall %s, fscore %s" % (args.threshold, fmt(res["precision"]),
                                                               fmt(res["recall"]), fmt(res["fscore"])))
    print("hausdorff %s" % fmt(res["hausdorff"]))
    print("  " + ", ".join("%s %.3f s" % kv for kv in phases.items()))
    return res


if __name__ == "__main__":
    main()
