#!/usr/bin/env python
"""bench_face_frame.py -- the per-frame work of the reference's camera_face_demo.py (:47-56) on the GPU.

For F faces (the face of the person fixture, 120 x 120 tiles pasted on a 640 x 480 procedural frame) the frame is
processed two ways with the seeded He weights of FaceNet:
  (a) host:   cv2.cvtColor, cv2.CascadeClassifier(haarcascade_frontalface_alt).detectMultiScale(gray, 1.2, 3,
              minSize=(1, 1)), then per face the demo's crop_face and FaceDetector.__call__ (one device pass per face);
  (b) device: FaceDetector.detect_frame(frame, CascadeClassifier(..., engine)) (opb_face_detect_frame, one call).
The cascade alone is timed both ways as well: cv2's detectMultiScale on the host CPU (with cv2's default thread count
and with one thread) against CascadeClassifier.detectMultiScale on the device (opb_cascade_detect).
Host wall clock around work that ends in a device synchronise (every device call synchronises before it returns),
after every shape has been warmed up; the variants alternate and the median of --reps repetitions is reported.

    python tools/bench_face_frame.py [--faces 1 4 16] [--reps 20] [--equal-tiles] [--out FILE]

--equal-tiles sets OPB_SMALL_BATCH=0 before any context is built, so batch 1 and batch n use the same conv tile shapes
and (a) and (b) must return bit-identical keypoints.  Prints one JSON line: GPU name, power limit and SM clocks read in
the same run, the host CPU and cv2's thread count, per-F median times, and whether (a) and (b) returned identical rects
and keypoints.  Needs an H100 and cv2 with its cascade files; there is no CPU path."""
import argparse
import json
import os
import statistics
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tools"), os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)
PKG = "chainer_realtime_multi-person_pose_estimation_b200"


def _frame(n_faces, tile):
    """640 x 480 procedural frame with n_faces copies of `tile` on a 5 x 4 grid of 128 x 120 cells"""
    import importlib
    frame = importlib.import_module(PKG + ".synthetic").procedural_image(480, 640, seed=5).copy()
    for i in range(n_faces):
        r, c = divmod(i, 5)
        frame[r * 120:r * 120 + 120, c * 128 + 4:c * 128 + 124] = tile
    return frame


def _crop_face(img, rect, scale):
    """crop_face of camera_face_demo.py:10-24"""
    h, w, _ = img.shape
    cx, cy = rect[0] + rect[2] / 2, rect[1] + rect[3] / 2
    cw, chh = rect[2] * scale, rect[3] * scale
    left, top = max(0, int(cx - cw / 2)), max(0, int(cy - chh / 2))
    right, bottom = min(w, int(cx + cw / 2)), min(h, int(cy + chh / 2))
    face = img[top:bottom, left:right]
    edge = np.max(face.shape[:-1])
    padded = np.zeros((edge, edge, face.shape[-1]), dtype=np.uint8)
    padded[0:face.shape[0], 0:face.shape[1]] = face
    return padded, (left, top)


def _bits(kps):
    return [None if k is None else (k[0], k[1], np.float32(k[2]).tobytes()) for k in kps]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--faces", type=int, nargs="+", default=[1, 4, 16])
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--equal-tiles", action="store_true")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if a.equal_tiles:
        os.environ["OPB_SMALL_BATCH"] = "0"
    import cv2
    import importlib
    from bench_whole_body import _gpu_info, _cpu_model
    from haar_ref import cascade_fixtures
    gpu_before = _gpu_info()
    pkg = importlib.import_module(PKG)
    fm = importlib.import_module(PKG + ".models.FaceNet")
    params = pkg.params
    net = fm.FaceNet()
    net.load_npz(pkg.synthetic.he_weights(0, layers=fm.LAYERS))
    det = pkg.FaceDetector(model=net, device=0)
    xml = os.path.join(cv2.data.haarcascades, "haarcascade_frontalface_alt.xml")
    host_cascade = cv2.CascadeClassifier(xml)
    dev_cascade = pkg.CascadeClassifier(xml, det.engine)
    f = cascade_fixtures()
    x, y, w, h = (int(v) for v in f["person_mn3_s1.2"][0])
    cx, cy = x + w // 2, y + h // 2
    tile = cv2.resize(f["person_bgr"][cy - 80:cy + 80, cx - 80:cx + 80], (120, 120), interpolation=cv2.INTER_AREA)
    threads = cv2.getNumThreads()

    def host(img):
        gray = cv2.cvtColor(img, cv2.COLOR_BGR2GRAY)
        rects = host_cascade.detectMultiScale(gray, scaleFactor=1.2, minNeighbors=3, minSize=(1, 1))
        order = sorted((tuple(int(v) for v in r) for r in rects), key=lambda r: (r[1], r[0], r[2], r[3]))
        res = []
        for r in order:
            crop, lt = _crop_face(img, r, params['face_crop_scale'])
            res.append((det(crop), lt))
        return order, res

    def device(img):
        rects, res = det.detect_frame(img, dev_cascade)
        return [tuple(int(v) for v in r) for r in (rects if len(rects) else [])], res

    def host_cascade_only(img):
        return host_cascade.detectMultiScale(cv2.cvtColor(img, cv2.COLOR_BGR2GRAY), 1.2, 3, minSize=(1, 1))

    def host_cascade_1t(img):
        cv2.setNumThreads(1)
        try:
            return host_cascade_only(img)
        finally:
            cv2.setNumThreads(threads)

    def device_cascade_only(img):
        return dev_cascade.detectMultiScale(img, 1.2, 3, (1, 1))

    variants = {"host_ms": host, "device_ms": device, "host_cascade_ms": host_cascade_only,
                "host_cascade_1thread_ms": host_cascade_1t, "device_cascade_ms": device_cascade_only}
    rows = []
    for n in a.faces:
        img = _frame(n, tile)
        for fn in variants.values():      # warm every shape and chunk of this frame
            fn(img)
            fn(img)
        times = {k: [] for k in variants}
        for _ in range(a.reps):
            for k, fn in variants.items():
                t0 = time.perf_counter()
                fn(img)
                times[k].append((time.perf_counter() - t0) * 1e3)
        hr, hres = host(img)
        dr, dres = device(img)
        same_kp = len(hres) == len(dres) and all(_bits(p[0]) == _bits(q[0]) and p[1] == q[1] for p, q in zip(hres, dres))
        rows.append(dict({k: round(statistics.median(v), 3) for k, v in times.items()}, faces_pasted=n,
                         faces_found=len(dr), rects_identical=hr == dr, keypoints_identical=bool(same_kp)))
    out = {"tool": "bench_face_frame", "frame": "640x480", "reps": a.reps, "equal_tiles": a.equal_tiles,
           "gpu": gpu_before, "gpu_after": _gpu_info(), "host_cpu": _cpu_model(), "cv2": cv2.__version__,
           "cv2_threads": threads, "rows": rows}
    line = json.dumps(out)
    print(line)
    if a.out:
        with open(a.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
