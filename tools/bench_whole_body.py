#!/usr/bin/env python
"""bench_whole_body.py -- the face / hand half of the reference's whole-body demo (demo.py:31-57) on the GPU.

For P synthetic people on a 640x480 procedural frame (stick figures of synthetic.person_layout, ~200 px tall), the face
box of PoseDetector.crop_face and the hand boxes of PoseDetector.crop_hands are derived from each pose, then timed two
ways with the seeded He weights of FaceNet and HandNet:
  (a) per crop: FaceDetector(crop_image(...)) once per face, HandDetector(...) once per hand, as demo.py does;
  (b) batched:  FaceDetector.detect_crops(frame, faces) once, HandDetector.detect_crops(frame, hands, types) once.
Host wall clock around work that ends in a device synchronise (every call of both variants synchronises before it
returns), after every shape has been warmed up; variants alternate, the median of --reps repetitions is reported.
The CocoPoseNet body pass of the same frame is timed once per run for scale.

    python tools/bench_whole_body.py [--people 1 4 8 16] [--reps 20] [--equal-tiles] [--out FILE]

--equal-tiles sets OPB_SMALL_BATCH=0 before any context is built, so batch 1 and batch n use the same conv tile shapes.
Prints one JSON line: GPU name, power limit and SM clocks read in the same run, per-P times, launch counts and whether
(a) and (b) returned identical keypoints.  Needs an H100; there is no CPU path."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
PKG = "chainer_realtime_multi-person_pose_estimation_b200"


def _gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=" + q, "--format=csv,noheader,nounits"],
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        return {"nvidia_smi_error": r.stdout.strip()[-200:]}
    name, pl, sm, sm_max = [v.strip() for v in r.stdout.strip().splitlines()[0].split(",")]
    return {"name": name, "power_limit_w": pl, "sm_clock_mhz": sm, "sm_clock_max_mhz": sm_max}


def _people(n):
    """[P,18,3] float poses (x, y, 1) of synthetic stick figures on the 640x480 frame"""
    import importlib
    syn = importlib.import_module(PKG + ".synthetic")
    xy = syn.person_layout(map_h=480, map_w=640, n_person=n, seed=n).astype(np.float64)
    return np.concatenate([xy, np.ones(xy.shape[:2] + (1,))], axis=2)


def _boxes(pose_det, frame, poses):
    faces, hands = [], []
    for pose in poses:
        pose = pose.copy()                     # crop_hands moves the hand joints in place (reference behaviour)
        unit = pose_det.get_unit_length(pose)
        img, bbox = pose_det.crop_face(frame, pose, unit)
        if img is not None and img.size:
            faces.append(bbox)
        hd = pose_det.crop_hands(frame, pose, unit)
        for side in ("left", "right"):
            if hd[side] is not None and hd[side]["img"].size:
                hands.append((hd[side]["bbox"], side))
    return faces, hands


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--people", type=int, nargs="+", default=[1, 4, 8, 16])
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--equal-tiles", action="store_true")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if a.equal_tiles:
        os.environ["OPB_SMALL_BATCH"] = "0"
    import torch
    if not torch.cuda.is_available():
        sys.exit("bench_whole_body.py needs an H100: no CUDA device (there is no CPU path)")
    import importlib
    pkg = importlib.import_module(PKG)
    syn, PD = pkg.synthetic, importlib.import_module(PKG + ".pose_detector")
    FD, HD = importlib.import_module(PKG + ".face_detector"), importlib.import_module(PKG + ".hand_detector")
    models = {k: importlib.import_module(PKG + ".models." + k) for k in ("CocoPoseNet", "FaceNet", "HandNet")}
    nets = {}
    for k, m in models.items():
        net = getattr(m, k)()
        net.load_npz(syn.he_weights(0, layers=getattr(m, "LAYERS", None)) if k != "CocoPoseNet" else syn.he_weights(0))
        nets[k] = net
    pose_det = PD.PoseDetector(model=nets["CocoPoseNet"], device=0)
    face_det = FD.FaceDetector(model=nets["FaceNet"], device=0)
    hand_det = HD.HandDetector(model=nets["HandNet"], device=0)
    frame = syn.procedural_image(480, 640, seed=5)
    crop = lambda b: pose_det.crop_image(frame, b)   # noqa: E731

    def per_crop(faces, hands):
        return ([face_det(crop(b)) for b in faces], [hand_det(crop(b), hand_type=t) for b, t in hands])

    def batched(faces, hands):
        return (face_det.detect_crops(frame, faces),
                hand_det.detect_crops(frame, [b for b, _ in hands], [t for _, t in hands]))

    def launches():
        return face_det.engine.launch_count() + hand_det.engine.launch_count()

    def bits(res):
        return [[None if k is None else (k[0], k[1], np.float32(k[2]).tobytes()) for k in kps] for part in res for kps in part]

    for _ in range(3):
        pose_det(frame)
    t0 = time.perf_counter()
    for _ in range(5):
        pose_det(frame)
    body_ms = (time.perf_counter() - t0) / 5 * 1e3
    gpu_before = _gpu_info()
    rows = []
    for p in a.people:
        faces, hands = _boxes(pose_det, frame, _people(p))
        for _ in range(2):                     # every chain shape of both variants
            per_crop(faces, hands)
            batched(faces, hands)
        l0 = launches(); ra = per_crop(faces, hands); la = launches() - l0
        l0 = launches(); rb = batched(faces, hands); lb = launches() - l0
        ba, bb = bits(ra), bits(rb)
        differ = sum(x != y for u, v in zip(ba, bb) for x, y in zip(u, v))
        ta, tb = [], []
        for _ in range(a.reps):
            t0 = time.perf_counter(); per_crop(faces, hands); ta.append(time.perf_counter() - t0)
            t0 = time.perf_counter(); batched(faces, hands); tb.append(time.perf_counter() - t0)
        rows.append({"people": p, "faces": len(faces), "hands": len(hands),
                     "per_crop_ms": round(float(np.median(ta)) * 1e3, 3), "batched_ms": round(float(np.median(tb)) * 1e3, 3),
                     "per_crop_ms_min": round(min(ta) * 1e3, 3), "batched_ms_min": round(min(tb) * 1e3, 3),
                     "speedup": round(float(np.median(ta) / np.median(tb)), 2),
                     "launches_per_crop": la, "launches_batched": lb,
                     "identical": ba == bb, "keypoints_differing": int(differ), "keypoints_total": sum(len(u) for u in ba)})
    res = {"tool": "bench_whole_body", "frame": "640x480", "precision": "comp", "equal_tiles": bool(a.equal_tiles),
           "reps": a.reps, "gpu": gpu_before, "gpu_after": _gpu_info(), "body_pass_ms": round(body_ms, 3), "rows": rows,
           "identical": all(r["identical"] for r in rows)}
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
