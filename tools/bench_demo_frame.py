#!/usr/bin/env python
"""bench_demo_frame.py -- the whole-body frame of the reference's demo.py (:24-57) on the GPU, two ways.

A 640 x 480 procedural frame with P injected stick-figure persons (synthetic.eight_person_lowres at the network-output
size; random weights cannot produce people), compensated precision, seeded He weights for CocoPoseNet, FaceNet and
HandNet:
  (a) chain:    the pose pass with the injected maps (resize_linear_u8 -> detect_batch(inject_*) -> _poses_from_records,
                what __call__ runs), the host helpers get_unit_length / crop_face / crop_hands per person,
                FaceDetector.detect_crops, HandDetector.detect_crops and draw_whole_body(..., engine=);
  (b) one call: whole_body.detect_whole_body (opb_whole_body_frame), the face and hand nets on their own streams.
Host wall clock around work that ends in a device synchronise (every call synchronises before it returns), after every
shape has been warmed up; (a) and (b) alternate and the median of --reps repetitions is reported, with the launches of
one frame and whether the two returned identical poses, boxes, keypoints and pictures.

    python tools/bench_demo_frame.py [--persons 1 4 8 16] [--reps 20] [--out FILE]

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


def _chain(pkg, pd, fd, hd, frame, in_hw, map_hw, d_paf, d_heat):
    """(a): today's best chain on the same injected maps"""
    wb = pkg.whole_body
    eng = pd.engine
    resized = eng.resize_linear_u8(frame, *in_hw)
    headers, persons = eng.detect_batch(resized[None], map_hw[0], map_hw[1], img_len=map_hw[1],
                                        inject_paf=d_paf.data_ptr(), inject_heat=d_heat.data_ptr())
    oh, ow = frame.shape[:2]
    poses, scores = pd._poses_from_records(headers[0], persons[0], ow / map_hw[1], oh / map_hw[0])
    boxes = []
    for pose in poses.copy():
        with np.errstate(all="ignore"):
            u = pd.get_unit_length(pose)
        if not np.isfinite(u):
            continue
        _, fb = pd.crop_face(frame, pose, u)
        hands = pd.crop_hands(frame, pose, u)
        for side, bb in (("face", fb), ("left", hands["left"] and hands["left"]["bbox"]),
                         ("right", hands["right"] and hands["right"]["bbox"])):
            if bb is not None and bb[2] > bb[0] and bb[3] > bb[1]:
                boxes.append((side, tuple(int(v) for v in bb)))
    faces = [b for s, b in boxes if s == "face"]
    hands = [(b, s) for s, b in boxes if s != "face"]
    fk = iter(fd.detect_crops(frame, faces) if faces else [])
    hk = iter(hd.detect_crops(frame, [b for b, _ in hands], [s for _, s in hands]) if hands else [])
    parts = [("face" if s == "face" else "hand", b, next(fk) if s == "face" else next(hk)) for s, b in boxes]
    picture = wb.draw_whole_body(frame, poses, parts, engine=eng)
    return poses, scores, parts, picture


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--persons", type=int, nargs="+", default=[1, 4, 8, 16])
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import importlib
    import torch
    from bench_whole_body import _gpu_info
    pkg = importlib.import_module(PKG)
    syn = pkg.synthetic
    gpu_before = _gpu_info()

    def net(kind):
        mod = importlib.import_module(PKG + ".models." + kind)
        m = getattr(mod, kind)()
        m.load_npz(syn.he_weights(0) if kind == "CocoPoseNet" else syn.he_weights(0, layers=mod.LAYERS))
        return m

    pd = pkg.PoseDetector(model=net("CocoPoseNet"), device=0, precision="comp")
    fd = pkg.FaceDetector(model=net("FaceNet"), device=0, precision="comp")
    hd = importlib.import_module(PKG + ".hand_detector").HandDetector(model=net("HandNet"), device=0, precision="comp")
    frame = syn.procedural_image(480, 640, seed=11)
    params = pkg.params
    in_w, in_h = pd.compute_optimal_size(frame, params["inference_img_size"])
    map_w, map_h = pd.compute_optimal_size(frame, params["heatmap_size"])
    dets = (pd, fd, hd)
    rows = []
    for P in a.persons:
        paf, heat = syn.eight_person_lowres(h=in_h // 8, w=in_w // 8, n_person=P, seed=0)
        d_paf = torch.from_numpy(np.ascontiguousarray(paf[None])).cuda()
        d_heat = torch.from_numpy(np.ascontiguousarray(heat[None])).cuda()
        torch.cuda.synchronize()
        run_a = lambda: _chain(pkg, pd, fd, hd, frame, (in_h, in_w), (map_h, map_w), d_paf, d_heat)   # noqa: E731
        run_b = lambda: pkg.whole_body._detect_whole_body(frame, pd, fd, hd, True, d_paf.data_ptr(),    # noqa: E731
                                                          d_heat.data_ptr())
        for _ in range(3):                                  # every chain shape of both paths built and warm
            ra, rb = run_a(), run_b()
        same = (np.array_equal(ra[0], rb[0]) and np.array_equal(ra[1], rb[1]) and
                [(k, b) for k, b, _ in ra[2]] == [(k, b) for k, b, _ in rb[2]] and
                all(x[2] == y[2] for x, y in zip(ra[2], rb[2])) and np.array_equal(ra[3], rb[4]))
        launches = []
        for fn in (run_a, run_b):
            before = sum(d.engine.launch_count() for d in dets)
            fn()
            launches.append(sum(d.engine.launch_count() for d in dets) - before)
        ta, tb = [], []
        for _ in range(a.reps):
            t0 = time.perf_counter(); run_a(); ta.append(time.perf_counter() - t0)
            t0 = time.perf_counter(); run_b(); tb.append(time.perf_counter() - t0)
        n_faces = sum(k == "face" for k, _, _ in rb[2])
        rows.append({"persons": P, "detected": int(len(rb[0])), "faces": n_faces, "hands": len(rb[2]) - n_faces,
                     "chain_ms": round(1e3 * statistics.median(ta), 3), "one_call_ms": round(1e3 * statistics.median(tb), 3),
                     "chain_ms_min": round(1e3 * min(ta), 3), "one_call_ms_min": round(1e3 * min(tb), 3),
                     "launches_chain": launches[0], "launches_one_call": launches[1], "identical": bool(same)})
        print(rows[-1], file=sys.stderr)
    res = {"bench": "demo_frame_640x480", "precision": "comp", "reps": a.reps, "rows": rows, "gpu": gpu_before,
           "gpu_after": _gpu_info()}
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
