"""Cases of the crop-box kernel of opb_whole_body_frame (csrc/whole_body.cuh), shared by the emulated CPU test and the
GPU test: person records in several families, run through Engine.test_whole_body_boxes and compared with the host
helpers PoseDetector.get_unit_length / crop_face / crop_hands on _poses_from_records' poses (a copy per person, as the
helpers move the hand joints in place).  Unit lengths must match bit for bit, boxes exactly, and the kept part list
must follow the skipping policy (no part for a non-finite unit length, no zero-width or zero-height box)."""
import numpy as np

from conftest import pkg

FRAME_SX, FRAME_SY = 640 / 432, 480 / 320      # a 640x480 frame: maps of 432x320
NOSE, NECK, R_ELBOW, R_HAND, L_ELBOW, L_HAND = 0, 1, 3, 4, 6, 7
BRANCH1 = (0, 1, 2, 5, 8, 11, 16, 17)           # the joints of limbs 14, 3, 0, 13, 9 (nose-neck, neck-waists, ...)


def _records(n):
    rec = np.zeros(n, pkg("_native").PERSON_DTYPE)
    rec["peak_id"] = -1
    return rec


def _put(rec, i, j, x, y):
    rec[i]["peak_id"][j] = j
    rec[i]["x"][j] = x
    rec[i]["y"][j] = y


def random_persons(rs, n, w=432, h=320):
    """joints present with a per-person probability, anywhere on a w x h map (border included)"""
    rec = _records(n)
    for i in range(n):
        p = rs.choice([0.15, 0.4, 0.7, 1.0])
        for j in range(18):
            if rs.rand() < p:
                _put(rec, i, j, rs.randint(0, w), rs.randint(0, h))
    return rec


def branch2_persons(rs, n, w=432, h=320):
    """limbs 14, 3, 0, 13, 9 all zero (their joints missing or on one point): the 19-ratio branch, often with 8 or more
    positive limbs (NumPy's pairwise sum)"""
    rec = _records(n)
    others = [j for j in range(18) if j not in BRANCH1]
    for i in range(n):
        if rs.rand() < 0.5:
            px, py = rs.randint(0, w), rs.randint(0, h)
            for j in BRANCH1:
                if rs.rand() < 0.7:
                    _put(rec, i, j, px, py)
        keep = rs.rand()
        for j in others:
            if rs.rand() < keep:
                _put(rec, i, j, rs.randint(0, w), rs.randint(0, h))
    return rec


def near_integer_persons(rs, n):
    """sx = sy = 1, neck present at the origin and the nose at a Pythagorean point (3k, 4k) with k a multiple of 17, so
    that u = fl(5k / 0.85) lies within an ulp of a multiple of 100: face edges, fl(u*1.2), fl(u*0.8) and fl(u*0.95) then
    sit on or one ulp from integers; hands on integer points, with and without the elbow"""
    rec = _records(n)
    for i in range(n):
        k = 17 * rs.randint(1, 6)
        _put(rec, i, NECK, 0, 0)
        _put(rec, i, NOSE, 3 * k * rs.choice([1, -1]) if rs.rand() < 0.2 else 3 * k, 4 * k)
        for hand, elbow in ((L_HAND, L_ELBOW), (R_HAND, R_ELBOW)):
            if rs.rand() < 0.8:
                _put(rec, i, hand, rs.randint(-50, 500), rs.randint(-50, 500))
            if rs.rand() < 0.3:
                _put(rec, i, elbow, rs.randint(0, 500), rs.randint(0, 500))
    return rec


def small_persons(rs, n):
    """the nose (or a hand) at or next to the origin and a short limb: negative edges near zero, which int() truncates
    toward zero, and with a small sx unit lengths below one pixel, i.e. zero-width boxes"""
    rec = _records(n)
    for i in range(n):
        _put(rec, i, NOSE, rs.randint(0, 3), rs.randint(0, 3))
        _put(rec, i, NECK, rs.randint(0, 4), rs.randint(0, 4))
        for hand in (L_HAND, R_HAND):
            if rs.rand() < 0.7:
                _put(rec, i, hand, rs.randint(0, 4), rs.randint(0, 4))
    return rec


def degenerate_persons(rs, n):
    """every present joint at the origin: no limb of positive length, unit length 0/0"""
    rec = _records(n)
    for i in range(n):
        for j in rs.choice(18, rs.randint(1, 6), replace=False):
            _put(rec, i, int(j), 0, 0)
    return rec


def reference(engine, rec, sx, sy):
    """(unit [n], boxes [n,3,4], present [n], kept parts [(person, side)]) from the host helpers"""
    native, PD = pkg("_native"), pkg("pose_detector")
    det = object.__new__(PD.PoseDetector)
    det.engine = engine
    det.crop_image = lambda img, bbox: np.zeros((max(bbox[3] - bbox[1], 0), max(bbox[2] - bbox[0], 0), 0), np.uint8)
    n = len(rec)
    header = np.zeros(1, native.HEADER_DTYPE)
    header["n_peaks"], header["n_persons"] = 1, n
    poses, _ = det._poses_from_records(header[0], rec, sx, sy)
    unit = np.full(n, np.nan)
    boxes = np.zeros((n, 3, 4), np.int64)
    present = np.zeros(n, np.int32)
    kept = []
    img = np.zeros((1, 1, 3), np.uint8)
    for i in range(n):
        pose = poses[i].copy()
        with np.errstate(all="ignore"):
            u = det.get_unit_length(pose)
        unit[i] = u
        if not np.isfinite(u):
            continue
        _, fb = det.crop_face(img, pose, u)
        hands = det.crop_hands(img, pose, u)
        for side, bb in enumerate((fb, hands["left"] and hands["left"]["bbox"], hands["right"] and hands["right"]["bbox"])):
            if bb is None:
                continue
            present[i] |= 1 << side
            boxes[i, side] = bb
            if bb[2] > bb[0] and bb[3] > bb[1]:
                kept.append((i, side))
    return unit, boxes, present, kept


def check(engine, rec, sx, sy):
    unit, boxes, present, parts = engine.test_whole_body_boxes(rec, sx, sy)
    r_unit, r_boxes, r_present, r_kept = reference(engine, rec, sx, sy)
    assert np.array_equal(np.isnan(unit), np.isnan(r_unit))
    fin = ~np.isnan(r_unit)
    assert np.array_equal(unit[fin].view(np.int64), r_unit[fin].view(np.int64)), "unit lengths differ"
    assert np.array_equal(present, r_present)
    for side in range(3):
        has = (present >> side & 1).astype(bool)
        assert np.array_equal(boxes[has, side], r_boxes[has, side]), "side %d boxes differ" % side
    assert [tuple(p) for p in parts] == r_kept
    return len(rec), int(fin.sum()), len(r_kept)


def run_cases(engine, scale=1):
    """every family at the 640x480 frame scale and at sx = sy = 1 (plus small scales for the sub-pixel unit lengths);
    returns the number of persons checked"""
    rs = np.random.RandomState(7)
    total = 0
    stats = {"skipped_unit": 0, "zero_box": 0, "branch2_8plus": 0}
    for sx, sy in ((FRAME_SX, FRAME_SY), (1.0, 1.0)):
        for fam in (random_persons, branch2_persons, small_persons, degenerate_persons):
            rec = fam(rs, 500 * scale)
            n, fin, _ = check(engine, rec, sx, sy)
            total += n
            stats["skipped_unit"] += n - fin
    total += check(engine, near_integer_persons(rs, 500 * scale), 1.0, 1.0)[0]
    for s in (0.1, 0.3, 0.45):
        rec = small_persons(rs, 300 * scale)
        u, b, present, parts = engine.test_whole_body_boxes(rec, s, s)
        stats["zero_box"] += int(sum(bin(int(p)).count("1") for p in present)) - len(parts)
        total += check(engine, rec, s, s)[0]
    rec = branch2_persons(rs, 300 * scale)
    check(engine, rec, 1.0, 1.0)
    total += len(rec)
    stats["branch2_8plus"] = int(sum(_positive_limbs(r) >= 8 for r in rec))
    assert stats["skipped_unit"] > 0 and stats["zero_box"] > 0 and stats["branch2_8plus"] > 0, stats
    return total, stats


def _positive_limbs(r):
    limbs = pkg("entity").params["limbs_point"]
    pt = [(float(r["x"][j]), float(r["y"][j])) if r["peak_id"][j] >= 0 else (0.0, 0.0) for j in range(18)]
    branch1 = [14, 3, 0, 13, 9]
    lens = [np.hypot(pt[b][0] - pt[a][0], pt[b][1] - pt[a][1]) for a, b in limbs]
    if any(lens[i] > 0 for i in branch1):
        return 0
    return sum(v > 0 for v in lens)


def check_out_of_range(engine):
    """a box edge beyond int32 is an error, never a converted value"""
    rec = _records(1)
    _put(rec, 0, NOSE, 1 << 30, 5)
    _put(rec, 0, NECK, 0, 5)
    try:
        engine.test_whole_body_boxes(rec, 4.0, 1.0)
    except pkg("_native").OpbError as e:
        assert "int32" in str(e)
    else:
        raise AssertionError("an out-of-range box edge was not reported")
