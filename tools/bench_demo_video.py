#!/usr/bin/env python
"""bench_demo_video.py -- the whole-body flow of the reference's demo.py (:24-57) on a batch of video frames, two ways.

N 640 x 480 procedural frames (a different seed per frame), each with P injected stick-figure persons
(synthetic.eight_person_lowres at the network-output size, a different seed per frame; random weights cannot produce
people), compensated precision, seeded He weights for CocoPoseNet, FaceNet and HandNet:
  (a) per frame: whole_body._detect_whole_body once per frame (opb_whole_body_frame: the pose pass at batch 1, the
      frame's crops through FaceNet / HandNet, the picture);
  (b) batch:     whole_body._detect_whole_body_batch on all N frames (opb_whole_body_batch: one pose forward at
      batch N, the crops of all frames in shared FaceNet / HandNet chunks, all pictures in one raster and one paint).
Host wall clock around work that ends in a device synchronise (every call synchronises before it returns), after every
shape of both paths has been warmed up; (a) and (b) alternate and the median of --reps repetitions is reported as
frames/s, with the launches of one batch and whether both returned identical poses, scores, parts, keypoints and
pictures.  --equal-tiles sets OPB_SMALL_BATCH=0 before any context is built (the same conv tile shapes at batch 1 and
batch N), under which the outputs must be identical bit for bit.

    python tools/bench_demo_video.py [--frames 4 8 16] [--persons 1 4 16] [--reps 10] [--equal-tiles] [--out FILE]

Prints one JSON line with the GPU name, power limit and SM clocks read in the same run.  Needs an H100."""
import argparse
import json
import os
import statistics
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)
PKG = "chainer_realtime_multi-person_pose_estimation_b200"


def _identical(ra, rb):
    """per-frame results of (a) and (b) equal bit for bit"""
    if len(ra) != len(rb):
        return False
    for a, b in zip(ra, rb):
        if not (np.array_equal(a[0], b[0]) and np.asarray(a[0]).shape == np.asarray(b[0]).shape and
                np.array_equal(a[1], b[1]) and a[3] == b[3] and np.array_equal(a[4], b[4])):
            return False
        if [(k, bb) for k, bb, _ in a[2]] != [(k, bb) for k, bb, _ in b[2]]:
            return False
        for (_, _, ka), (_, _, kb) in zip(a[2], b[2]):
            for p, q in zip(ka, kb):
                if (p is None) != (q is None):
                    return False
                if p is not None and (p[0] != q[0] or p[1] != q[1] or
                                      np.float32(p[2]).tobytes() != np.float32(q[2]).tobytes()):
                    return False
    return True


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, nargs="+", default=[4, 8, 16])
    ap.add_argument("--persons", type=int, nargs="+", default=[1, 4, 16])
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--equal-tiles", action="store_true")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if a.equal_tiles:
        os.environ["OPB_SMALL_BATCH"] = "0"              # read when a context or chain is built: set before any
    import importlib
    import torch
    from bench_whole_body import _gpu_info
    pkg = importlib.import_module(PKG)
    syn, wb = pkg.synthetic, pkg.whole_body
    gpu_before = _gpu_info()

    def net(kind):
        mod = importlib.import_module(PKG + ".models." + kind)
        m = getattr(mod, kind)()
        m.load_npz(syn.he_weights(0) if kind == "CocoPoseNet" else syn.he_weights(0, layers=mod.LAYERS))
        return m

    pd = pkg.PoseDetector(model=net("CocoPoseNet"), device=0, precision="comp")
    fd = pkg.FaceDetector(model=net("FaceNet"), device=0, precision="comp")
    hd = importlib.import_module(PKG + ".hand_detector").HandDetector(model=net("HandNet"), device=0, precision="comp")
    dets = (pd, fd, hd)
    params = pkg.params
    probe = syn.procedural_image(480, 640, seed=0)
    in_w, in_h = pd.compute_optimal_size(probe, params["inference_img_size"])
    cases = {}
    for N in a.frames:
        frames = np.stack([syn.procedural_image(480, 640, seed=100 + f) for f in range(N)])
        for P in a.persons:
            maps = [syn.eight_person_lowres(h=in_h // 8, w=in_w // 8, n_person=P, seed=f) for f in range(N)]
            d_paf = torch.from_numpy(np.ascontiguousarray(np.stack([m[0] for m in maps]))).cuda()
            d_heat = torch.from_numpy(np.ascontiguousarray(np.stack([m[1] for m in maps]))).cuda()
            cases[(N, P)] = (frames, d_paf, d_heat)
    torch.cuda.synchronize()

    def run_a(c):
        frames, d_paf, d_heat = c
        return [wb._detect_whole_body(frames[f], pd, fd, hd, True, d_paf[f].data_ptr(), d_heat[f].data_ptr())
                for f in range(len(frames))]

    def run_b(c):
        frames, d_paf, d_heat = c
        return wb._detect_whole_body_batch(frames, pd, fd, hd, True, d_paf.data_ptr(), d_heat.data_ptr())

    for _ in range(2):                                      # every chain shape of both paths built and warm
        for c in cases.values():
            run_a(c)
            run_b(c)
    rows = []
    for (N, P), c in cases.items():
        ra, rb = run_a(c), run_b(c)
        launches = []
        for fn in (run_a, run_b):
            before = sum(d.engine.launch_count() for d in dets)
            fn(c)
            launches.append(sum(d.engine.launch_count() for d in dets) - before)
        ta, tb = [], []
        for _ in range(a.reps):
            t0 = time.perf_counter(); run_a(c); ta.append(time.perf_counter() - t0)
            t0 = time.perf_counter(); run_b(c); tb.append(time.perf_counter() - t0)
        ma, mb = statistics.median(ta), statistics.median(tb)
        n_parts = sum(len(r[2]) for r in rb)
        n_faces = sum(k == "face" for r in rb for k, _, _ in r[2])
        rows.append({"frames": N, "persons": P, "detected": int(sum(len(r[0]) for r in rb)), "faces": n_faces,
                     "hands": n_parts - n_faces, "per_frame_fps": round(N / ma, 1), "batch_fps": round(N / mb, 1),
                     "per_frame_ms": round(1e3 * ma, 3), "batch_ms": round(1e3 * mb, 3),
                     "speedup": round(ma / mb, 3), "launches_per_frame_calls": launches[0],
                     "launches_batch": launches[1], "identical": bool(_identical(ra, rb))})
        print(rows[-1], file=sys.stderr)
    res = {"bench": "demo_video_640x480", "precision": "comp", "equal_tiles": bool(a.equal_tiles), "reps": a.reps,
           "rows": rows, "gpu": gpu_before, "gpu_after": _gpu_info()}
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
