"""`-m gpu`: whole_body.detect_whole_body (opb_whole_body_frame) against the chain a user strings together today --
pose_detector(img), the host crop helpers per person, FaceDetector / HandDetector.detect_crops and the host
draw_whole_body -- on 640x480 frames: noise persons from random weights, injected stick figures, an empty frame.
Poses, scores, boxes, keypoints and the picture must be equal bit for bit.  Also: the crop-box kernel's hook cases on the
device (nvcc contracts a*b + c unless told not to), draw=False, draw_last_result afterwards, the launch count, and
every argument error raised with nothing launched."""
import numpy as np
import pytest

import whole_body_cases as W
from conftest import pkg

pytestmark = pytest.mark.gpu


def _model(kind):
    mod = pkg("models.FaceNet" if kind == "face" else "models.HandNet")
    m = getattr(mod, "FaceNet" if kind == "face" else "HandNet")()
    m.load_npz(pkg("synthetic").he_weights(0, layers=mod.LAYERS))
    return m


@pytest.fixture(scope="module")
def dets():
    PD = pkg("pose_detector")
    model = pkg("models.CocoPoseNet").CocoPoseNet()
    model.load_npz(pkg("synthetic").he_weights(0))
    return (PD.PoseDetector(model=model, device=0), pkg("face_detector").FaceDetector(model=_model("face"), device=0),
            pkg("hand_detector").HandDetector(model=_model("hand"), device=0))


def _launches(*ds):
    return sum(d.engine.launch_count() for d in ds)


def _expected_parts(pose_det, img, poses):
    """the demo's boxes in its order under the skipping policy: no part for a non-finite unit length, none for an empty
    box; crop_hands moves the hand joints of its argument, so each person is a copy"""
    out = []
    for i, pose in enumerate(np.asarray(poses).reshape(-1, 18, 3)):
        pose = pose.copy()
        with np.errstate(all="ignore"):
            u = pose_det.get_unit_length(pose)
        if not np.isfinite(u):
            continue
        _, fb = pose_det.crop_face(img, pose, u)
        hands = pose_det.crop_hands(img, pose, u)
        for side, bb in (("face", fb), ("left", hands["left"] and hands["left"]["bbox"]),
                         ("right", hands["right"] and hands["right"]["bbox"])):
            if bb is not None and bb[2] > bb[0] and bb[3] > bb[1]:
                out.append((i, side, tuple(int(v) for v in bb)))
    return out


def _compare(dets, frame, poses, scores, got, mismatch_label=""):
    """got = detect_whole_body's result; the reference chain starts from (poses, scores)"""
    pose_det, face, hand = dets
    g_poses, g_scores, parts, owners, picture = got
    assert np.array_equal(g_poses, poses) and g_poses.shape == np.asarray(poses).shape
    assert np.array_equal(g_scores, scores)
    exp = _expected_parts(pose_det, frame, poses)
    assert [(o[0], o[1], p[1]) for o, p in zip(owners, parts)] == exp
    assert all(k == ("face" if s == "face" else "hand") for (k, _, _), (_, s) in zip(parts, owners))
    assert all(type(v) is int for _, b, _ in parts for v in b)
    faces = [b for _, s, b in exp if s == "face"]
    hands = [(b, s) for _, s, b in exp if s != "face"]
    fk = face.detect_crops(frame, faces) if faces else []
    hk = hand.detect_crops(frame, [b for b, _ in hands], [s for _, s in hands]) if hands else []
    ref_kps = iter(fk), iter(hk)
    want = [next(ref_kps[0]) if s == "face" else next(ref_kps[1]) for _, s, _ in exp]
    bad = sum(a != b for (_, _, a), b in zip(parts, want))
    print("%s%d poses, %d faces, %d hands, %d keypoint lists differ from detect_crops"
          % (mismatch_label, len(poses), len(faces), len(hands), bad))
    assert bad == 0
    ref_pic = pkg("whole_body").draw_whole_body(frame, poses, parts)
    assert np.array_equal(picture, ref_pic), "%d pixels differ" % int((picture != ref_pic).any(2).sum())
    return len(faces), len(hands)


def test_box_kernel_on_device(dets):
    total, stats = W.run_cases(dets[0].engine)
    print("whole-body boxes on the device: %d persons, %s" % (total, stats))
    W.check_out_of_range(dets[0].engine)


@pytest.mark.parametrize("seed", [3, 5])
def test_noise_persons_640x480(dets, seed):
    pose_det, face, hand = dets
    wb = pkg("whole_body")
    frame = pkg("synthetic").procedural_image(480, 640, seed=seed)
    poses, scores = pose_det(frame)
    got = wb.detect_whole_body(frame, pose_det, face, hand)
    nf, nh = _compare(dets, frame, poses, scores, got, "seed %d: " % seed)
    assert len(poses) and nf and nh, "random-weight maps give some 'persons'; an empty flow tests nothing"


def _stick_figures(pose_det, frame, n_person, seed=0):
    """device maps of n_person stick figures at the network-output size of the frame, and the reference chain's
    (poses, scores): resize_linear_u8 -> detect_batch(inject_*) -> _poses_from_records"""
    import torch
    params = pkg("entity").params
    in_w, in_h = pose_det.compute_optimal_size(frame, params["inference_img_size"])
    map_w, map_h = pose_det.compute_optimal_size(frame, params["heatmap_size"])
    paf, heat = pkg("synthetic").eight_person_lowres(h=in_h // 8, w=in_w // 8, n_person=n_person, seed=seed)
    d_paf = torch.from_numpy(np.ascontiguousarray(paf[None])).cuda()
    d_heat = torch.from_numpy(np.ascontiguousarray(heat[None])).cuda()
    torch.cuda.synchronize()
    eng = pose_det.engine
    resized = eng.resize_linear_u8(frame, in_h, in_w)
    headers, persons = eng.detect_batch(resized[None], map_h, map_w, img_len=map_w, inject_paf=d_paf.data_ptr(),
                                        inject_heat=d_heat.data_ptr())
    oh, ow = frame.shape[:2]
    poses, scores = pose_det._poses_from_records(headers[0], persons[0], ow / map_w, oh / map_h)
    return (d_paf, d_heat), poses, scores


@pytest.mark.parametrize("n_person", [1, 4, 8, 16])
def test_stick_figures_640x480(dets, n_person):
    pose_det, face, hand = dets
    wb = pkg("whole_body")
    frame = pkg("synthetic").procedural_image(480, 640, seed=11)
    (d_paf, d_heat), poses, scores = _stick_figures(pose_det, frame, n_person)
    got = wb._detect_whole_body(frame, pose_det, face, hand, True, d_paf.data_ptr(), d_heat.data_ptr())
    nf, nh = _compare(dets, frame, poses, scores, got, "%d stick figures: " % n_person)
    assert len(poses) >= n_person and nf and nh        # 16 figures on a 62x46 map group into a few more persons


def test_empty_frame(dets):
    """zero maps: no peaks, no persons, no parts; the picture is addWeighted(img, 0.6, img, 0.4, 0) == img"""
    import torch
    pose_det, face, hand = dets
    frame = pkg("synthetic").procedural_image(480, 640, seed=2)
    z_paf = torch.zeros((1, 38, 46, 62), dtype=torch.float32, device="cuda")
    z_heat = torch.zeros((1, 19, 46, 62), dtype=torch.float32, device="cuda")
    before = _launches(face, hand)
    poses, scores, parts, owners, picture = pkg("whole_body")._detect_whole_body(
        frame, pose_det, face, hand, True, z_paf.data_ptr(), z_heat.data_ptr())
    assert len(poses) == 0 and len(scores) == 0 and parts == [] and owners == []
    assert _launches(face, hand) == before                       # neither net runs without crops
    assert np.array_equal(picture, pkg("whole_body").draw_whole_body(frame, poses, []))
    assert np.array_equal(picture, frame)


def test_draw_false_and_draw_last_result(dets):
    pose_det, face, hand = dets
    wb = pkg("whole_body")
    frame = pkg("synthetic").procedural_image(480, 640, seed=3)
    full = wb.detect_whole_body(frame, pose_det, face, hand)
    after = pose_det.draw_last_result(frame)
    poses, scores, parts, owners, picture = wb.detect_whole_body(frame, pose_det, face, hand, draw=False)
    assert picture is None
    assert np.array_equal(poses, full[0]) and np.array_equal(scores, full[1]) and owners == full[3]
    assert [(k, b) for k, b, _ in parts] == [(k, b) for k, b, _ in full[2]]
    assert all(a[2] == b[2] for a, b in zip(parts, full[2]))
    # the pose context holds this frame's result
    assert np.array_equal(after, pkg("pose_detector").draw_person_pose(frame, full[0]))


def test_launch_count(dets):
    """pose pass of __call__ + 1 box kernel + each net's detect_crops launches + the picture: records -> poses (with
    persons), raster (with persons or parts), paint"""
    pose_det, face, hand = dets
    wb = pkg("whole_body")
    frame = pkg("synthetic").procedural_image(480, 640, seed=5)
    wb.detect_whole_body(frame, pose_det, face, hand)             # every chain shape built
    l0 = pose_det.engine.launch_count()
    poses, _ = pose_det(frame)
    n_pose = pose_det.engine.launch_count() - l0
    exp = _expected_parts(pose_det, frame, poses)
    faces = [b for _, s, b in exp if s == "face"]
    hands = [(b, s) for _, s, b in exp if s != "face"]
    f0 = face.engine.launch_count()
    face.detect_crops(frame, faces)
    n_face = face.engine.launch_count() - f0
    h0 = hand.engine.launch_count()
    hand.detect_crops(frame, [b for b, _ in hands], [s for _, s in hands])
    n_hand = hand.engine.launch_count() - h0
    n_draw = int(len(poses) > 0) + int(len(poses) > 0 or len(exp) > 0) + 1
    before = [d.engine.launch_count() for d in dets]
    wb.detect_whole_body(frame, pose_det, face, hand)
    got = [d.engine.launch_count() - b for d, b in zip(dets, before)]
    assert got == [n_pose + 1 + n_draw, n_face, n_hand], (got, n_pose, n_face, n_hand, n_draw)
    before = [d.engine.launch_count() for d in dets]
    wb.detect_whole_body(frame, pose_det, face, hand, draw=False)
    got = [d.engine.launch_count() - b for d, b in zip(dets, before)]
    assert got == [n_pose + 1, n_face, n_hand]


def test_errors_launch_nothing(dets):
    pose_det, face, hand = dets
    native, wb = pkg("_native"), pkg("whole_body")
    frame = pkg("synthetic").procedural_image(480, 640, seed=3)

    def nothing_launched(fn, exc):
        before = [d.engine.launch_count() for d in dets]
        with pytest.raises(exc):
            fn()
        assert [d.engine.launch_count() for d in dets] == before

    nothing_launched(lambda: wb.detect_whole_body(frame, pose_det, hand, face), ValueError)      # swapped slots
    nothing_launched(lambda: wb.detect_whole_body(frame, face, pose_det, hand), ValueError)
    nothing_launched(lambda: wb.detect_whole_body(frame[..., 0], pose_det, face, hand), ValueError)
    pose_det.precise = True
    try:
        nothing_launched(lambda: wb.detect_whole_body(frame, pose_det, face, hand), ValueError)
    finally:
        pose_det.precise = False
    face.engine.device = 1                 # a detector on another device (checked before any device work)
    try:
        nothing_launched(lambda: wb.detect_whole_body(frame, pose_det, face, hand), ValueError)
    finally:
        face.engine.device = 0
    pe = pose_det.engine
    # the C entry refuses the same, and bad sizes, before anything is enqueued
    for args in ((hand.engine, face.engine, frame, 368, 496, 320, 432), (face.engine, hand.engine, frame, 368, 490, 320, 432),
                 (face.engine, hand.engine, frame, 368, 496, 0, 432)):
        nothing_launched(lambda: pe.whole_body_frame(*args, 432, 368, 0.1, 368, 0.1), native.OpbError)
    nothing_launched(lambda: pe.whole_body_frame(face.engine, hand.engine, frame, 368, 496, 320, 432, 432, 36, 0.1, 368,
                                                 0.1), native.OpbError)
    nothing_launched(lambda: face.engine.whole_body_frame(face.engine, hand.engine, frame, 368, 496, 320, 432, 432, 368,
                                                          0.1, 368, 0.1), native.OpbError)


def test_record_status_raises_as_call(dets):
    """a result status (here: more persons than max_persons) raises what __call__ raises"""
    _, face, hand = dets
    PD = pkg("pose_detector")
    model = pkg("models.CocoPoseNet").CocoPoseNet()
    model.load_npz(pkg("synthetic").he_weights(0))
    small = PD.PoseDetector(model=model, device=0, max_persons=1)
    frame = pkg("synthetic").procedural_image(480, 640, seed=3)
    with pytest.raises(pkg("_native").OpbError) as e_call:
        small(frame)
    with pytest.raises(pkg("_native").OpbError):
        pkg("whole_body").detect_whole_body(frame, small, face, hand)
    print("status error:", e_call.value)
