"""`-m gpu`: the Haar cascade on the device (csrc/cascade.cuh, opb_cascade_detect) and the camera-face frame
(opb_face_detect_frame).

(1) every window's result code and final stage sum equal the NumPy restatement (tests/haar_ref.py) bit for bit;
(2) CascadeClassifier.detectMultiScale equals cv2's recorded outputs (tests/golden/cascade_outputs.npz) on every
    fixture frame (tests/golden/cascade_*.png) and case, for gray and BGR input, and cv2 live for the default and eye
    cascades where cv2 is importable;
(3) FaceDetector.detect_frame equals camera_face_demo.py's loop -- its crop_face, then FaceDetector.__call__ on each
    padded crop -- bit for bit with OPB_SMALL_BATCH=0, in parity and compensated precision, including faces at the
    right and bottom borders and a frame of 20 faces (two forward chunks);
(4) launch counts, and errors that return before anything is launched."""
import ctypes as C
import functools
import os

import numpy as np
import pytest

from conftest import pkg
import haar_ref as H
import test_gpu_keypoints as K  # noqa: E402  (plain helpers; the gpu mark belongs to that module only)

pytestmark = pytest.mark.gpu

NAMES = ("person", "dinner", "people")


def _haar_dir():
    try:
        import cv2
    except ImportError:
        return None
    d = getattr(getattr(cv2, "data", None), "haarcascades", "")
    return d if os.path.isfile(os.path.join(d, "haarcascade_frontalface_alt.xml")) else None


def _xml(name):
    d = _haar_dir()
    if d is None:
        pytest.skip("cv2.data.haarcascades (haarcascade_%s.xml) is not available" % name)
    return os.path.join(d, "haarcascade_%s.xml" % name)


@functools.lru_cache(None)
def frames():
    pytest.importorskip("cv2")         # decodes the PNG fixtures
    return H.cascade_fixtures()


@functools.lru_cache(None)
def classifier(name="frontalface_alt"):
    return pkg("cascade").CascadeClassifier(_xml(name))


def _rows(rects):
    return [tuple(int(v) for v in r) for r in (rects if len(rects) else [])]


@pytest.mark.parametrize("frame,sf", [("person", 1.2), ("dinner", 1.1), ("people", 1.3)])
def test_windows_bit_exact(frame, sf):
    cc = classifier()
    gray = frames()[frame + "_gray"]
    codes, sums = cc.engine.test_cascade_windows(gray, sf, (1, 1))
    ref_c, ref_s = [], []
    for layer in H.pyramid(gray, cc.tables.window, sf, (1, 1)):
        ys, xs = H.layer_windows(cc.tables, layer)
        c, s = H.eval_windows(cc.tables, layer, ys, xs)
        ref_c.append(c)
        ref_s.append(s)
    ref_c, ref_s = np.concatenate(ref_c), np.concatenate(ref_s)
    assert codes.shape == ref_c.shape
    assert np.array_equal(codes, ref_c)
    assert np.array_equal(sums.view(np.int64), ref_s.view(np.int64))
    # BGR input converts on the device to the same gray frame
    codes_bgr, sums_bgr = cc.engine.test_cascade_windows(frames()[frame + "_bgr"], sf, (1, 1))
    assert np.array_equal(codes_bgr, codes) and np.array_equal(sums_bgr.view(np.int64), sums.view(np.int64))


def test_recorded_outputs_gray_and_bgr():
    mk = pytest.importorskip("oracle.make_cascade_goldens")
    cc = classifier()
    f = frames()
    for name in NAMES:
        for key, (sf, mn, mins, maxs) in mk.CASES.items():
            want = _rows(f["%s_%s" % (name, key)])
            for kind in ("gray", "bgr"):
                got = cc.detectMultiScale(f["%s_%s" % (name, kind)], sf, mn, mins, maxs)
                assert _rows(got) == want, (name, key, kind)
                if len(want):
                    assert got.dtype == np.int32 and got.shape == (len(want), 4)
                else:
                    assert got == ()


def test_cv2_live_other_cascades_and_frames():
    cv2 = pytest.importorskip("cv2")
    f = frames()
    g = f["person_gray"]
    cases = [g, np.ascontiguousarray(g[:301, :457]), np.ascontiguousarray(g[37:, 11:]), g[:19, :40].copy(),
             np.full((120, 160), 128, np.uint8)]
    for name in ("frontalface_alt", "frontalface_default", "eye"):
        cc = classifier(name)
        ref = cv2.CascadeClassifier(_xml(name))
        for img in cases:
            for mn in (0, 3):
                want = H.sort_rects(ref.detectMultiScale(img, 1.2, mn, minSize=(1, 1)))
                assert _rows(cc.detectMultiScale(img, 1.2, mn, (1, 1))) == want, (name, img.shape, mn)


# ---- camera_face_demo.py's frame ---------------------------------------------------------------------------------
def demo_crop_face(img, rect):
    """crop_face of camera_face_demo.py:10-24 (right / bottom clamp to w / h; zero padding to a square)."""
    params = pkg("entity").params
    h, w, _ = img.shape
    cx, cy = rect[0] + rect[2] / 2, rect[1] + rect[3] / 2
    cw, chh = rect[2] * params['face_crop_scale'], rect[3] * params['face_crop_scale']
    left, top = max(0, int(cx - cw / 2)), max(0, int(cy - chh / 2))
    right, bottom = min(w, int(cx + cw / 2)), min(h, int(cy + chh / 2))
    face = img[top:bottom, left:right]
    edge = np.max(face.shape[:-1])
    padded = np.zeros((edge, edge, face.shape[-1]), dtype=np.uint8)
    padded[0:face.shape[0], 0:face.shape[1]] = face
    return padded, (left, top)


def demo_loop(det, cascade, img):
    """camera_face_demo.py:47-56 with this package's cascade and FaceDetector.__call__"""
    gray = H.bgr_to_gray(img)
    rects = cascade.detectMultiScale(gray, scaleFactor=1.2, minNeighbors=3, minSize=(1, 1))
    out = []
    for r in (rects if len(rects) else []):
        crop, lt = demo_crop_face(img, r)
        out.append((det(crop), lt))
    return rects, out


def _same_keypoints(a, b):
    assert len(a) == len(b)
    for ka, kb in zip(a, b):
        assert (ka is None) == (kb is None), (ka, kb)
        if ka is not None:
            assert type(ka[0]) is int and type(ka[1]) is int and isinstance(ka[2], np.float32)
            assert (ka[0], ka[1]) == (kb[0], kb[1]) and ka[2].tobytes() == np.float32(kb[2]).tobytes(), (ka, kb)


def _face_tile():
    """The person fixture's face with a margin, 160 x 160."""
    f = frames()
    x, y, w, h = _rows(f["person_mn3_s1.2"])[0]
    cx, cy = x + w // 2, y + h // 2
    return f["person_bgr"][cy - 80:cy + 80, cx - 80:cx + 80]


def _demo_frames():
    f = frames()
    bgr = f["person_bgr"]
    x, y, w, h = _rows(f["person_mn3_s1.2"])[0]
    right = np.ascontiguousarray(bgr[:, :x + w + 4])            # the padded crop reaches past the right edge
    bottom = np.ascontiguousarray(bgr[:y + h + 3, :])           # ... and past the bottom edge
    tile = _face_tile()
    many = np.ascontiguousarray(np.tile(tile, (4, 5, 1)))       # 20 faces: a chunk of 16 and one of 4
    return {"person": bgr, "dinner": f["dinner_bgr"], "right": right, "bottom": bottom, "many": many}


@pytest.mark.parametrize("precision", ["parity", "comp"])
def test_detect_frame_equals_demo_loop(precision, monkeypatch):
    monkeypatch.setenv("OPB_SMALL_BATCH", "0")        # equal conv tile shapes at batch 1 and batch n
    det = pkg("face_detector").FaceDetector(model=K._model("face"), device=0, precision=precision)
    cascade = pkg("cascade").CascadeClassifier(_xml("frontalface_alt"), det.engine)
    counts = {}
    for name, img in _demo_frames().items():
        rects, res = det.detect_frame(img, cascade)
        ref_rects, ref_res = demo_loop(det, cascade, img)
        assert _rows(rects) == _rows(ref_rects), name
        assert len(res) == len(ref_res) == len(_rows(rects))
        for (kp, lt), (rkp, rlt) in zip(res, ref_res):
            assert lt == rlt, name
            _same_keypoints(kp, rkp)
        counts[name] = len(res)
    assert counts["person"] >= 1 and counts["many"] > 16, counts
    # the right / bottom cases pad past the frame edge
    for name in ("right", "bottom"):
        img = _demo_frames()[name]
        for r in _rows(det.detect_frame(img, cascade)[0]):
            crop, (l, t) = demo_crop_face(img, r)
            assert l + crop.shape[1] > img.shape[1] or t + crop.shape[0] > img.shape[0]


def test_launch_counts_and_errors(monkeypatch):
    det = pkg("face_detector").FaceDetector(model=K._model("face"), device=0, precision="parity")
    cascade = pkg("cascade").CascadeClassifier(_xml("frontalface_alt"), det.engine)
    eng = det.engine
    img = frames()["person_bgr"]
    cascade.detectMultiScale(img, 1.2, 3, (1, 1))                   # plan and tables for this shape
    l0 = eng.launch_count()
    rects = cascade.detectMultiScale(img, 1.2, 3, (1, 1))
    assert eng.launch_count() - l0 == 5                              # pyramid, row scan, column scan, windows, compaction
    boxes = [(int(x), int(y), int(x + w), int(y + h)) for x, y, w, h in rects]
    det.detect_crops(img, boxes)
    l0 = eng.launch_count()
    det.detect_crops(img, boxes)
    crops_launches = eng.launch_count() - l0
    l0 = eng.launch_count()
    det.detect_frame(img, cascade)
    assert eng.launch_count() - l0 == 5 + crops_launches

    # errors return before anything is launched
    lib, ctx = eng.lib, eng.ctx
    a = np.ascontiguousarray(img)
    out = np.empty((16, 4), np.int32)
    n = C.c_int(0)

    def call(h=a.shape[0], w=a.shape[1], ch=3, sf=1.2, mn=3, mins=(1, 1), maxs=(0, 0), cap=16):
        return lib.opb_cascade_detect(ctx, C.c_void_p(a.ctypes.data), 0, h, w, ch, sf, mn, mins[0], mins[1], maxs[0],
                                      maxs[1], C.c_void_p(out.ctypes.data), cap, C.byref(n))

    l0 = eng.launch_count()
    for kw in ({"sf": 1.0}, {"sf": 0.5}, {"sf": float("nan")}, {"mn": -1}, {"mins": (-1, 1)}, {"maxs": (0, -5)},
               {"ch": 0}, {"ch": 2}, {"h": 0}, {"cap": -1}):
        assert call(**kw) == pkg("_native").ERR_ARG, kw
    assert eng.launch_count() == l0
    with pytest.raises(ValueError):
        cascade.detectMultiScale(img, 1.0)
    with pytest.raises(ValueError):
        cascade.detectMultiScale(img.astype(np.float32))
    assert call(cap=0) == pkg("_native").ERR_CAPACITY and n.value == 1
    # a frame smaller than the window: nothing found, nothing launched
    l0 = eng.launch_count()
    assert cascade.detectMultiScale(img[:19, :19].copy(), 1.2, 3) == ()
    assert eng.launch_count() == l0
    # a context without FaceNet refuses the frame call
    pose_cascade = pkg("cascade").CascadeClassifier(_xml("frontalface_alt"))
    with pytest.raises(pkg("_native").OpbError):
        pose_cascade.engine.face_detect_frame(img, 1.2, 3, (1, 1), (0, 0), 1.5, 368, 0.1)
