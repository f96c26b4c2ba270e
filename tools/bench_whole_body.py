#!/usr/bin/env python
"""bench_whole_body.py -- the face / hand half of the reference's whole-body demo (demo.py:31-57) on the GPU.

For P synthetic people on a 640x480 procedural frame (stick figures of synthetic.person_layout, ~200 px tall), the face
box of PoseDetector.crop_face and the hand boxes of PoseDetector.crop_hands are derived from each pose, then timed two
ways with the seeded He weights of FaceNet and HandNet:
  (a) per crop: FaceDetector(crop_image(...)) once per face, HandDetector(...) once per hand, as demo.py does;
  (b) batched:  FaceDetector.detect_crops(frame, faces) once, HandDetector.detect_crops(frame, hands, types) once.
The result picture of demo.py (the blended skeleton of the P poses, then per person the face, left hand and right hand
keypoints of (b) with their boxes) is composed two ways as well:
  (c) host:   whole_body.draw_whole_body(frame, poses, parts), i.e. the cv2 calls demo.py makes;
  (d) device: the same with engine= (opb_draw_whole_body: one upload, two launches, one download).
Host wall clock around work that ends in a device synchronise (every device call synchronises before it returns),
after every shape has been warmed up; variants alternate, the median of --reps repetitions is reported.
The CocoPoseNet body pass of the same frame is timed once per run for scale.  (c) runs on the host CPU, whose model
the result records next to the GPU's.

    python tools/bench_whole_body.py [--people 1 4 8 16] [--reps 20] [--equal-tiles] [--out FILE]

--equal-tiles sets OPB_SMALL_BATCH=0 before any context is built, so batch 1 and batch n use the same conv tile shapes.
Prints one JSON line: GPU name, power limit and SM clocks read in the same run, the host CPU model, per-P times, launch
counts, whether (a) and (b) returned identical keypoints and whether (c) and (d) drew identical images.  Needs an H100;
there is no CPU path."""
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


def _cpu_model():
    """the host CPU's model name (lscpu, else /proc/cpuinfo) and its logical CPU count: the host composition runs on it"""
    import platform
    name = None
    try:
        r = subprocess.run(["lscpu"], stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
        name = next((ln.split(":", 1)[1].strip() for ln in r.stdout.splitlines() if ln.startswith("Model name")), None)
    except OSError:
        pass
    if not name:
        try:
            with open("/proc/cpuinfo") as f:
                name = next((ln.split(":", 1)[1].strip() for ln in f if ln.startswith("model name")), None)
        except OSError:
            pass
    return "%s (%s, %d logical CPUs)" % (name or "model not reported", platform.machine(), os.cpu_count() or 0)


def _people(n):
    """[P,18,3] float poses (x, y, 1) of synthetic stick figures on the 640x480 frame"""
    import importlib
    syn = importlib.import_module(PKG + ".synthetic")
    xy = syn.person_layout(map_h=480, map_w=640, n_person=n, seed=n).astype(np.float64)
    return np.concatenate([xy, np.ones(xy.shape[:2] + (1,))], axis=2)


def _boxes(pose_det, frame, poses):
    """face boxes, (hand box, side) pairs, and the demo's drawing order: ("face" | "hand", index into faces / hands)"""
    faces, hands, order = [], [], []
    for pose in poses:
        pose = pose.copy()                     # crop_hands moves the hand joints in place (reference behaviour)
        unit = pose_det.get_unit_length(pose)
        img, bbox = pose_det.crop_face(frame, pose, unit)
        if img is not None and img.size:
            order.append(("face", len(faces)))
            faces.append(bbox)
        hd = pose_det.crop_hands(frame, pose, unit)
        for side in ("left", "right"):
            if hd[side] is not None and hd[side]["img"].size:
                order.append(("hand", len(hands)))
                hands.append((hd[side]["bbox"], side))
    return faces, hands, order


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
    WB = importlib.import_module(PKG + ".whole_body")
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
        poses = _people(p)
        faces, hands, order = _boxes(pose_det, frame, poses)
        for _ in range(2):                     # every chain shape of both variants
            per_crop(faces, hands)
            batched(faces, hands)
        l0 = launches(); ra = per_crop(faces, hands); la = launches() - l0
        l0 = launches(); rb = batched(faces, hands); lb = launches() - l0
        ba, bb = bits(ra), bits(rb)
        differ = sum(x != y for u, v in zip(ba, bb) for x, y in zip(u, v))
        parts = [("face", faces[i], rb[0][i]) if k == "face" else ("hand", hands[i][0], rb[1][i]) for k, i in order]
        eng = pose_det.engine
        host_img = WB.draw_whole_body(frame, poses, parts)
        l0 = eng.launch_count(); dev_img = WB.draw_whole_body(frame, poses, parts, engine=eng); ld = eng.launch_count() - l0
        ta, tb, tc, td = [], [], [], []
        for _ in range(a.reps):
            t0 = time.perf_counter(); per_crop(faces, hands); ta.append(time.perf_counter() - t0)
            t0 = time.perf_counter(); batched(faces, hands); tb.append(time.perf_counter() - t0)
        for _ in range(a.reps):
            t0 = time.perf_counter(); WB.draw_whole_body(frame, poses, parts); tc.append(time.perf_counter() - t0)
            t0 = time.perf_counter(); WB.draw_whole_body(frame, poses, parts, engine=eng); td.append(time.perf_counter() - t0)
        rows.append({"people": p, "faces": len(faces), "hands": len(hands),
                     "per_crop_ms": round(float(np.median(ta)) * 1e3, 3), "batched_ms": round(float(np.median(tb)) * 1e3, 3),
                     "per_crop_ms_min": round(min(ta) * 1e3, 3), "batched_ms_min": round(min(tb) * 1e3, 3),
                     "speedup": round(float(np.median(ta) / np.median(tb)), 2),
                     "launches_per_crop": la, "launches_batched": lb,
                     "identical": ba == bb, "keypoints_differing": int(differ), "keypoints_total": sum(len(u) for u in ba),
                     "compose_host_ms": round(float(np.median(tc)) * 1e3, 3),
                     "compose_device_ms": round(float(np.median(td)) * 1e3, 3),
                     "compose_speedup": round(float(np.median(tc) / np.median(td)), 2),
                     "launches_compose_device": ld, "images_identical": bool(np.array_equal(host_img, dev_img))})
    res = {"tool": "bench_whole_body", "frame": "640x480", "precision": "comp", "equal_tiles": bool(a.equal_tiles),
           "reps": a.reps, "gpu": gpu_before, "gpu_after": _gpu_info(), "host_cpu": _cpu_model(),
           "body_pass_ms": round(body_ms, 3), "rows": rows,
           "identical": all(r["identical"] for r in rows), "images_identical": all(r["images_identical"] for r in rows)}
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
