"""`-m gpu`: FaceDetector.detect_crops / HandDetector.detect_crops (opb_keypoints_detect_crops) -- every face or hand
crop of a frame in one batched device pass.

(1) the four keypoint goldens pasted into one frame meet the criteria of
    test_gpu_keypoints.py::test_detector_end_to_end_parity, in parity and compensated precision;
(2) with OPB_SMALL_BATCH=0 (the same conv tile shapes at batch 1 and batch n) ~40 mixed crops over three forward
    chunks equal the per-crop path bit for bit;
(3) the demo's whole-body flow (demo.py:31-57) on PoseDetector output: batched == per-person loop;
(4) errors: pose context, empty crops; n = 0."""
import numpy as np
import pytest

from conftest import load_golden, pkg
from oracle import restate as R
import test_gpu_keypoints as K  # noqa: E402  (plain helpers; the gpu mark belongs to that module only)

pytestmark = pytest.mark.gpu


def _detectors(precision=None):
    kw = {} if precision is None else {"precision": precision}
    return (pkg("face_detector").FaceDetector(model=K._model("face"), device=0, **kw),
            pkg("hand_detector").HandDetector(model=K._model("hand"), device=0, **kw))


def _crop(img, bbox):
    return pkg("pose_detector").PoseDetector.crop_image(None, img, bbox)


def _mismatches(a, b):
    """number of keypoints of list a that differ from list b in validity, x, y or the float32 confidence bits"""
    assert len(a) == len(b)
    bad = 0
    for ka, kb in zip(a, b):
        if (ka is None) != (kb is None):
            bad += 1
        elif ka is not None:
            assert type(ka[0]) is int and type(ka[1]) is int and isinstance(ka[2], np.float32)
            bad += (ka[0], ka[1]) != (kb[0], kb[1]) or np.float32(ka[2]).tobytes() != np.float32(kb[2]).tobytes()
    return bad


# golden -> (left, top) in a 480 x 640 frame: face_401x401 touches the top-left corner, the left hand the bottom-right
PLACES = {"face_401x401_he0.npz": (0, 0), "face_150x170_he0.npz": (420, 10), "hand_120x131_he0_right.npz": (420, 200),
          "hand_120x131_he0_left.npz": (509, 360)}


@pytest.mark.parametrize("precision", ["parity", "comp"])
def test_goldens_in_one_frame(precision):
    import cv2
    face, hand = _detectors(precision)
    frame = np.zeros((480, 640, 3), np.uint8)
    cases = []
    for name, kind, hand_type in K.CASES:
        g = load_golden(name)
        h, w, seed = (int(v) for v in g["img_hw_seed"])
        left, top = PLACES[name]
        frame[top:top + h, left:left + w] = pkg("synthetic").procedural_image(h, w, seed=seed)
        cases.append((name, kind, hand_type, g, (left, top, left + w, top + h)))
    faces = [c for c in cases if c[1] == "face"]
    hands = [c for c in cases if c[1] == "hand"]
    got = dict(zip([c[0] for c in faces], face.detect_crops(frame, [c[4] for c in faces])))
    got.update(zip([c[0] for c in hands], hand.detect_crops(frame, [c[4] for c in hands], [c[2] for c in hands])))
    for name, kind, hand_type, g, bbox in cases:
        det = face if kind == "face" else hand
        img = _crop(frame, bbox)
        src = cv2.flip(img, 1) if hand_type == "left" else img
        err = float(np.abs(det.model(R.keypoint_preprocess(cv2.resize(src, (368, 368))))[-1][0] - g["heat_lo"]).max())
        assert err <= K.MAP_TOL
        ref = K._golden_list(g)
        sm = R.gaussian_smooth(np.ascontiguousarray(K._oracle_maps(g, hand_type)[:-1], np.float32))
        eps = K.TIE_FACTOR * max(err, 1e-6)
        flips = 0
        for c, (a, b) in enumerate(zip(got[name], ref)):
            mx = float(sm[c].max())
            if (a is None) != (b is None):
                assert abs(mx - np.float32(0.1)) < eps, "channel %d validity differs with margin %.3e" % (c, mx - 0.1)
                flips += 1
                continue
            if a is None:
                continue
            assert abs(float(a[2]) - float(b[2])) <= K.MAP_TOL
            if (a[0], a[1]) != (b[0], b[1]):
                assert mx - float(sm[c][a[1], a[0]]) < eps, "channel %d argmax differs beyond the near-tie margin" % c
                flips += 1
        print("%s %s-precision batched: near-tie flips %d of %d" % (name, precision, flips, len(ref)))
        assert flips <= (3 if precision == "parity" else 6)


def _mixed_crops(rs, n, fh, fw):
    """n boxes cycling through: inside, partly outside, fully outside, 368 x 368, larger than 368, small"""
    out = []
    for i in range(n):
        kind = i % 6
        if kind == 0:
            h, w = rs.randint(60, 250, 2); t, l = rs.randint(0, fh - h), rs.randint(0, fw - w)
        elif kind == 1:
            h, w = rs.randint(80, 300, 2); t, l = rs.randint(-h // 2, fh - h // 2), rs.choice([-w // 3, fw - 2 * w // 3])
        elif kind == 2:
            # below or right of the frame by more than the crop's own size: crop_image's slicing is then empty on both
            # sides (a box ending at a negative row or column would wrap around in its NumPy slices instead)
            h, w = rs.randint(30, 200, 2)
            if i % 4:
                t, l = fh + h + rs.randint(0, 20), rs.randint(0, fw - w)
            else:
                t, l = rs.randint(0, fh - h), fw + w + rs.randint(0, 20)
        elif kind == 3:
            h = w = 368; t, l = rs.randint(-40, fh - 300), rs.randint(-40, fw - 300)
        elif kind == 4:
            h, w = rs.randint(369, 520, 2); t, l = rs.randint(-60, 100), rs.randint(-60, 200)
        else:
            h, w = rs.randint(3, 24, 2); t, l = rs.randint(0, fh), rs.randint(0, fw)
        out.append((int(l), int(t), int(l + w), int(t + h)))
    return out


def test_batched_equals_per_crop_bit_for_bit(monkeypatch):
    monkeypatch.setenv("OPB_SMALL_BATCH", "0")        # equal conv tile shapes at batch 1 and batch n
    face, hand = _detectors()
    rs = np.random.RandomState(7)
    frame = pkg("synthetic").procedural_image(480, 640, seed=12)
    boxes = _mixed_crops(rs, 40, 480, 640)
    types = ["left" if i % 2 else ("right" if i % 4 else "other") for i in range(len(boxes))]
    eng = hand.engine
    l0 = eng.launch_count()
    got = hand.detect_crops(frame, boxes, types)
    l40 = eng.launch_count() - l0
    l0 = eng.launch_count()
    got16 = hand.detect_crops(frame, boxes[:16], types[:16])
    l16 = eng.launch_count() - l0
    bad = 0
    for b, t, kps in zip(boxes, types, got):
        bad += _mismatches(kps, hand(_crop(frame, b), hand_type=t))
    assert got16 == got[:16]
    l0 = eng.launch_count()
    hand(_crop(frame, (0, 0, 368, 368)))                  # no resize launch at 368 x 368
    chain = eng.launch_count() - l0 - 4                   # ... upsample, two smoothing passes, arg-max
    # 40 crops = chunks of 16 + 16 + 8: per chunk crop-resize, chain, upsample; then smoothing x2 and arg-max once
    assert l16 == chain + 5 and l40 == 3 * (chain + 2) + 3, (l16, l40, chain)
    fboxes = boxes[::2]
    fgot = face.detect_crops(frame, fboxes)
    for b, kps in zip(fboxes, fgot):
        bad += _mismatches(kps, face(_crop(frame, b)))
    print("hand crops %d (%d launches), face crops %d: %d keypoints differ" % (len(boxes), l40, len(fboxes), bad))
    assert bad == 0


def _whole_body_crops(frame):
    """PoseDetector on a procedural frame (random weights: many noise 'persons'), then get_unit_length / crop_face /
    crop_hands per pose (demo.py:31-57) -> face boxes, hand boxes and hand types in the demo's order"""
    PD = pkg("pose_detector")
    model = pkg("models.CocoPoseNet").CocoPoseNet()
    model.load_npz(pkg("synthetic").he_weights(0))
    pose = PD.PoseDetector(model=model, device=0)
    poses, _ = pose(frame)
    faces, hands = [], []
    with np.errstate(all="ignore"):
        for person_pose in poses:
            try:
                unit = pose.get_unit_length(person_pose)
                img, bbox = pose.crop_face(frame, person_pose, unit)
                hd = pose.crop_hands(frame, person_pose, unit)
            except (ValueError, IndexError, OverflowError):   # degenerate noise poses (no limb to measure)
                continue
            if img is not None and img.size:
                faces.append(bbox)
            for side in ("left", "right"):
                if hd[side] is not None and hd[side]["img"].size:
                    hands.append((hd[side]["bbox"], side))
    return faces, hands


def test_demo_whole_body_flow(monkeypatch):
    frame = pkg("synthetic").procedural_image(480, 640, seed=3)
    faces, hands = _whole_body_crops(frame)
    print("demo flow: %d face crops, %d hand crops" % (len(faces), len(hands)))
    assert faces and hands, "random-weight maps give some 'persons'; an empty demo flow tests nothing"

    def run():
        face, hand = _detectors()
        per = ([face(_crop(frame, b)) for b in faces], [hand(_crop(frame, b), hand_type=t) for b, t in hands])
        bat = (face.detect_crops(frame, faces), hand.detect_crops(frame, [b for b, _ in hands], [t for _, t in hands]))
        return (sum(_mismatches(a, b) for a, b in zip(bat[0], per[0])) +
                sum(_mismatches(a, b) for a, b in zip(bat[1], per[1])))

    default_bad = run()
    print("demo flow, default settings: %d keypoint entries differ bit for bit between batched and per-crop" % default_bad)
    monkeypatch.setenv("OPB_SMALL_BATCH", "0")
    assert run() == 0


def test_errors_and_empty_call():
    native = pkg("_native")
    face, hand = _detectors("fast")
    frame = np.zeros((64, 80, 3), np.uint8)
    assert face.detect_crops(frame, []) == [] and hand.detect_crops(frame, [], []) == []
    l0 = face.engine.launch_count()
    for bad in ([(5, 5, 5, 20)], [(0, 0, 10, 10), (3, 9, 20, 4)], [(1, 2, 3)], [(0.5, 0, 10, 10)]):
        with pytest.raises(ValueError):
            face.detect_crops(frame, bad)
    with pytest.raises(ValueError):
        hand.detect_crops(frame, [(0, 0, 10, 10)], ["left", "right"])
    table = np.zeros(1, native.CROP_DTYPE)
    table[0] = (4, 4, 4, 12, 0, 0)
    with pytest.raises(native.OpbError, match="-2"):
        face.engine.keypoints_detect_crops(frame, table, 368, 0.1)
    assert face.engine.launch_count() == l0
    model = pkg("models.CocoPoseNet").CocoPoseNet()
    model.load_npz(pkg("synthetic").he_weights(0))
    pose_eng = pkg("pose_detector").PoseDetector(model=model, device=0).engine
    with pytest.raises(native.OpbError, match="-3"):
        pose_eng.keypoints_detect_crops(frame, [(0, 0, 10, 10)], 368, 0.1)
