"""`-m gpu`: whole_body.draw_whole_body with engine= (opb_draw_whole_body, csrc/overlay.cuh) against the host path, the
cv2 calls of demo.py:28-57 -- addWeighted of the skeleton overlay, then per part draw_face_keypoints /
draw_hand_keypoints and cv2.rectangle.  Every case requires the device image to equal the host image bit for bit.

The test bodies are plain functions of an `engine`, so tests/test_emu_draw_whole_body.py runs them under the CPU
emulation too; the demo flow (PoseDetector -> crops -> detect_crops -> picture on a 640x480 frame) runs here only."""
import numpy as np
import pytest

from conftest import pkg

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def engine():
    return pkg("_native").Engine(0, pkg("pose_detector").make_opb_params())


def _same(engine, img, poses, parts):
    wb = pkg("whole_body")
    ref = wb.draw_whole_body(img, poses, parts)
    got = wb.draw_whole_body(img, poses, parts, engine=engine)
    assert got.shape == ref.shape and got.dtype == ref.dtype
    assert np.array_equal(got, ref), "%d pixels differ" % int((got != ref).any(2).sum())
    return ref


def _random_poses(rs, n, h, w):
    """float [n,18,3] poses with every present joint inside the image, some on its border"""
    poses = np.zeros((n, 18, 3), np.float64)
    for p in range(n):
        cx, cy = rs.uniform(0, w - 1), rs.uniform(0, h - 1)
        for j in range(18):
            if rs.rand() < 0.2:
                continue
            x = np.clip(cx + rs.normal(0, w / 6.0), 0, w - 1)
            y = np.clip(cy + rs.normal(0, h / 6.0), 0, h - 1)
            if rs.rand() < 0.2:
                x = rs.choice([0, w - 1])
            poses[p, j] = (x, y, 2)
    return poses


def _random_part(rs, kind, h, w, where):
    """(kind, bbox, keypoints) with the box inside, partly outside or entirely outside an h x w frame; keypoints
    inside the box, just outside it, on or just past the frame border, far away, or absent"""
    n = 70 if kind == "face" else 21
    bw, bh = (int(v) for v in rs.randint(3, 90, 2))
    if where == "inside":
        l, t = rs.randint(0, max(1, w - bw)), rs.randint(0, max(1, h - bh))
    elif where == "partly":
        l, t = rs.choice([-bw // 2, w - bw // 2, rs.randint(0, w)]), rs.choice([-bh // 2, h - bh // 2, rs.randint(0, h)])
    else:
        l, t = rs.choice([-bw - rs.randint(1, 40), w + rs.randint(0, 40)]), rs.randint(-bh, h + bh)
    l, t = int(l), int(t)
    kps = []
    for _ in range(n):
        if rs.rand() < 0.15:
            kps.append(None)
            continue
        x, y = int(rs.randint(-6, bw + 6)), int(rs.randint(-6, bh + 6))
        r = rs.rand()
        if r < 0.15:
            x = int(rs.choice([-l, w - 1 - l, -l - 1, w - l]))
        elif r < 0.3:
            y = int(rs.choice([-t, h - 1 - t, -t - 1, h - t]))
        elif r < 0.35:
            x, y = int(rs.randint(-400, 400)), int(rs.randint(-400, 400))
        kps.append([x, y, np.float32(rs.rand())])
    return kind, (l, t, l + bw, t + bh), kps


def test_random_frames_skeletons_and_parts(engine):
    """frames of several sizes (odd, narrow, one pixel wide), skeletons under faces and hands inside, partly and
    entirely outside the frame"""
    rs = np.random.RandomState(11)
    sizes = [(120, 160, 3, 6), (97, 61, 2, 9), (33, 200, 1, 5), (240, 17, 2, 4), (64, 64, 4, 12), (1, 90, 0, 3),
             (70, 1, 0, 3), (240, 320, 5, 10)]
    for h, w, n_poses, n_parts in sizes:
        img = rs.randint(0, 256, (h, w, 3)).astype(np.uint8)
        poses = _random_poses(rs, n_poses, h, w)
        parts = [_random_part(rs, rs.choice(["face", "hand"]), h, w, ("inside", "partly", "outside")[k % 3])
                 for k in range(n_parts)]
        _same(engine, img, poses, parts)


def _polyline_part(kind, bbox, path):
    """a part whose first len(path) keypoints form `path` (crop coordinates); face: contour 0..16, hand: thumb 0..4"""
    n = 70 if kind == "face" else 21
    kps = [None] * n
    for k, (x, y) in enumerate(path):
        kps[k] = [x, y, np.float32(0.5)]
    return kind, bbox, kps


# zero-length, horizontal, vertical, 45 degrees, steep, shallow, leftwards, upwards, and long segments leaving the box
_FACE_PATH = [(0, 0), (0, 0), (12, 0), (12, 12), (24, 24), (27, 50), (70, 54), (40, 54), (20, 40), (18, 2), (-30, -20),
              (90, -3), (91, 60), (-5, 61), (30, 30), (31, 29), (29, 31)]
_HAND_PATH = [(10, 10), (10, 10), (40, 11), (39, 60), (-20, -45)]


def test_segment_directions_and_clipping(engine):
    """1-px lines in every direction class, walked from either end, at offsets that put them inside the frame, across
    each frame edge and corner, and wholly outside it"""
    h, w = 57, 83
    rs = np.random.RandomState(5)
    img = rs.randint(0, 256, (h, w, 3)).astype(np.uint8)
    for l, t in [(5, 5), (-40, 3), (60, -20), (-10, 40), (50, 30), (-100, -100), (-60, -50), (20, 50), (70, 10)]:
        parts = [_polyline_part("face", (l, t, l + 60, t + 55), _FACE_PATH),
                 _polyline_part("hand", (l + 3, t + 4, l + 40, t + 50), _HAND_PATH),
                 _polyline_part("face", (l, t, l + 60, t + 55), [(x, -y) for x, y in _FACE_PATH]),
                 _polyline_part("hand", (l, t, l + 30, t + 30), [(-x, y) for x, y in _HAND_PATH])]
        _same(engine, img, np.zeros((0, 18, 3)), parts)
    # random 1-px lines with both ends far outside a small frame: clipLine decides every pixel
    for _ in range(8):
        path = [(int(rs.randint(-150, 150)), int(rs.randint(-150, 150))) for _ in range(17)]
        _same(engine, img, np.zeros((0, 18, 3)), [_polyline_part("face", (20, 20, 40, 40), path)])


def test_overlapping_parts_overwrite_in_order(engine):
    """parts drawn over each other and over the skeleton: the order of the list decides the pixels"""
    h, w = 80, 96
    rs = np.random.RandomState(9)
    img = rs.randint(0, 256, (h, w, 3)).astype(np.uint8)
    poses = _random_poses(rs, 3, h, w)
    parts = []
    for k in range(6):
        kind = ("face", "hand")[k % 2]
        n = 70 if kind == "face" else 21
        kps = [[int(rs.randint(0, 30)), int(rs.randint(0, 30)), np.float32(0.5)] for _ in range(n)]
        parts.append((kind, (20 + k, 15 + k, 60 - k, 55 - k), kps))
    a = _same(engine, img, poses, parts)
    b = _same(engine, img, poses, parts[::-1])
    assert not np.array_equal(a, b), "the overlap is too small to test the overwrite order"


def _blend_case():
    """a frame whose pixels under each skeleton colour take every value 0..255: 9 one-joint poses per joint colour, one
    two-joint pose per drawn limb; returns (img, poses, {colour index: pixels whose last primitive has it})"""
    import cv2
    limbs = [tuple(int(v) for v in ab) for ab in pkg("entity").params["limbs_point"]]
    h, w = 136, 200
    img = np.zeros((h, w, 3), np.uint8)
    poses, cover = [], {}
    for j in range(18):
        base = 0
        for k in range(9):
            cell = j * 9 + k
            cx, cy = 4 + 8 * (cell % 11), 4 + 8 * (cell // 11)
            pose = np.zeros((18, 3))
            pose[j] = (cx, cy, 2)
            poses.append(pose)
            m = np.zeros((h, w), np.uint8)
            cv2.circle(m, (cx, cy), 3, 1, -1)
            ys, xs = np.nonzero(m)
            img[ys, xs] = ((base + np.arange(len(ys))) % 256)[:, None]
            base += len(ys)
            cover.setdefault(("joint", j), []).extend(img[ys, xs, 0].tolist())
    for r, l in enumerate([l for l in range(19) if l not in (9, 13)]):
        ja, jb = limbs[l]
        y, x0, x1 = 4 + 8 * r, 96, 196
        pose = np.zeros((18, 3))
        pose[ja], pose[jb] = (x0, y, 2), (x1, y, 2)
        poses.append(pose)
        m = np.zeros((h, w), np.uint8)
        cv2.line(m, (x0, y), (x1, y), 1, 2)
        cv2.circle(m, (x0, y), 3, 0, -1)
        cv2.circle(m, (x1, y), 3, 0, -1)
        ys, xs = np.nonzero(m)
        img[ys, xs] = (np.arange(len(ys)) % 256)[:, None]
        cover[("limb", l)] = img[ys, xs, 0].tolist()
    return img, np.array(poses), cover


def test_blend_every_value_under_every_skeleton_colour(engine):
    """addWeighted(img, 0.6, skeleton, 0.4, 0) for every uint8 frame value under each of the 17 drawn limb colours and
    18 joint colours (their components are 0, 85, 170 and 255 in every channel)"""
    img, poses, cover = _blend_case()
    assert len(cover) == 35 and all(set(v) == set(range(256)) for v in cover.values())
    ref = _same(engine, img, poses, [])
    assert (ref != img).any(), "the skeleton must change the frame"


def test_empty_poses_and_parts(engine):
    """no poses (both empty shapes): the frame with only the parts drawn; no parts: the blended skeleton; neither: the
    frame itself"""
    wb, fd, hd = pkg("whole_body"), pkg("face_detector"), pkg("hand_detector")
    import cv2
    rs = np.random.RandomState(2)
    h, w = 61, 77
    img = rs.randint(0, 256, (h, w, 3)).astype(np.uint8)
    parts = [_random_part(rs, "face", h, w, "partly"), _random_part(rs, "hand", h, w, "inside")]
    only_parts = img.copy()
    for kind, bbox, kps in parts:
        only_parts = (fd.draw_face_keypoints if kind == "face" else hd.draw_hand_keypoints)(only_parts, kps, bbox[:2])
        cv2.rectangle(only_parts, bbox[:2], bbox[2:], (255, 255, 255), 1)
    for empty in (np.zeros((0, 18, 3)), np.array([])):
        assert np.array_equal(_same(engine, img, empty, parts), only_parts)
        assert np.array_equal(_same(engine, img, empty, []), img)
    poses = _random_poses(rs, 2, h, w)
    skel = _same(engine, img, poses, [])
    assert np.array_equal(skel, cv2.addWeighted(img, 0.6, pkg("pose_detector").draw_person_pose(img, poses), 0.4, 0))
    original = img.copy()
    wb.draw_whole_body(img, poses, parts, engine=engine)
    assert np.array_equal(img, original), "the input frame must not be modified"


def test_errors_and_launch_count(engine):
    """ValueError before any launch for an unknown kind, a keypoint count that does not match the kind or a malformed
    box; OpbError (OPB_ERR_ARG) for a coordinate above 2^20 in magnitude and a present joint outside the image; two
    launches per call (raster, paint), one when there is nothing to draw"""
    wb, native = pkg("whole_body"), pkg("_native")
    rs = np.random.RandomState(4)
    h, w = 40, 50
    img = rs.randint(0, 256, (h, w, 3)).astype(np.uint8)
    face = _random_part(rs, "face", h, w, "inside")
    hand = _random_part(rs, "hand", h, w, "partly")
    l0 = engine.launch_count()
    for bad in ([("foot", face[1], face[2])], [("face", face[1], face[2][:69])], [("hand", hand[1], face[2])],
                [("hand", hand[1], hand[2] + [None])], [("face", (0, 0, 10), face[2])], [("face", (0.5, 0, 9, 9), face[2])],
                [("hand", (0, 0, 2 ** 31, 9), hand[2])], [face, ("face",)]):
        with pytest.raises(ValueError):
            wb.draw_whole_body(img, np.zeros((0, 18, 3)), bad, engine=engine)
    big = 2 ** 20 + 1
    far_point = list(hand[2])
    far_point[3] = [big - hand[1][0] + 1, 0, np.float32(0.5)]
    out_joint = np.zeros((1, 18, 3))
    out_joint[0, 4] = (w, 3, 2)
    for poses, parts in ((np.zeros((0, 18, 3)), [("face", (big, 0, big + 5, 5), face[2])]),
                         (np.zeros((0, 18, 3)), [("hand", (0, -big, 5, 5), hand[2])]),
                         (np.zeros((0, 18, 3)), [face, ("hand", hand[1], far_point)]),
                         (out_joint, [face])):
        with pytest.raises(native.OpbError, match="-2"):
            wb.draw_whole_body(img, poses, parts, engine=engine)
    # the C entry point refuses an unknown kind and a point table that is too short
    table = np.zeros(1, native.PART_DTYPE)
    pts = np.zeros((21, 3), np.int32)
    for kind, n_points in ((7, 21), (native.PART_FACE, 21)):
        table[0] = (kind, 0, 0, 5, 5, 0)
        out = np.empty_like(img)
        rc = engine.lib.opb_draw_whole_body(engine.ctx, native._ptr(img), native.OPB_HOST, h, w, None, 0,
                                            native._ptr(table), 1, native._ptr(pts), n_points, native._ptr(out),
                                            native.OPB_HOST)
        assert rc == native.ERR_ARG
    assert engine.launch_count() == l0
    # launches per call
    poses = _random_poses(rs, 2, h, w)
    for poses_, parts, n in ((poses, [face, hand], 2), (poses, [], 2), (np.zeros((0, 18, 3)), [hand], 2),
                             (np.zeros((0, 18, 3)), [], 1)):
        l0 = engine.launch_count()
        wb.draw_whole_body(img, poses_, parts, engine=engine)
        assert engine.launch_count() - l0 == n


def _demo_parts(pose_det, frame, poses):
    """demo.py:31-57: per person the face box, then the left and the right hand box, with the detectors' keypoints
    of every crop from one detect_crops call per net"""
    boxes = []
    with np.errstate(all="ignore"):
        for person_pose in poses.copy():            # crop_hands moves the hand joints in place (reference behaviour)
            try:
                unit = pose_det.get_unit_length(person_pose)
                img, bbox = pose_det.crop_face(frame, person_pose, unit)
                hd = pose_det.crop_hands(frame, person_pose, unit)
            except (ValueError, IndexError, OverflowError):   # degenerate noise poses (no limb to measure)
                continue
            if img is not None and img.size:
                boxes.append(("face", bbox, None))
            for side in ("left", "right"):
                if hd[side] is not None and hd[side]["img"].size:
                    boxes.append(("hand", hd[side]["bbox"], side))
    return boxes


def test_demo_flow_640x480():
    """PoseDetector on a procedural 640x480 frame (random weights: many noise 'persons') -> crop_face / crop_hands ->
    FaceDetector / HandDetector.detect_crops -> draw_whole_body: device == host"""
    import test_gpu_keypoints as K
    PD = pkg("pose_detector")
    model = pkg("models.CocoPoseNet").CocoPoseNet()
    model.load_npz(pkg("synthetic").he_weights(0))
    pose_det = PD.PoseDetector(model=model, device=0)
    face = pkg("face_detector").FaceDetector(model=K._model("face"), device=0)
    hand = pkg("hand_detector").HandDetector(model=K._model("hand"), device=0)
    frame = pkg("synthetic").procedural_image(480, 640, seed=3)
    poses, _ = pose_det(frame)
    boxes = _demo_parts(pose_det, frame, poses)
    faces = [b for k, b, _ in boxes if k == "face"]
    hands = [(b, s) for k, b, s in boxes if k == "hand"]
    assert len(poses) and faces and hands, "random-weight maps give some 'persons'; an empty demo flow tests nothing"
    fk = iter(face.detect_crops(frame, faces))
    hk = iter(hand.detect_crops(frame, [b for b, _ in hands], [s for _, s in hands]))
    parts = [(k, b, next(fk) if k == "face" else next(hk)) for k, b, _ in boxes]
    print("demo flow: %d poses, %d faces, %d hands" % (len(poses), len(faces), len(hands)))
    ref = _same(pose_det.engine, frame, poses, parts)
    assert not np.array_equal(ref, frame)
