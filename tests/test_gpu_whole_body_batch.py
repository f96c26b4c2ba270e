"""`-m gpu`: whole_body.detect_whole_body_batch (opb_whole_body_batch) on batches of 640x480 frames against
detect_whole_body per frame and against the step-by-step chain.
  - N = 1 under the default policy is detect_whole_body bit for bit, launch counts included;
  - with OPB_SMALL_BATCH=0 (the same conv tile shapes at batch 1 and batch N) every frame of a batch equals
    detect_whole_body on that frame alone: poses, scores, parts, owners, keypoints and picture;
  - under the default policy (N = 8) poses and scores equal PoseDetector.detect_batch, parts the host helpers and
    pictures the host draw_whole_body; keypoint lists that differ from per-frame detect_crops (other chunk tile shapes)
    are counted, not asserted;
  - the launch count, draw=False, and every argument error raised with nothing launched."""
import numpy as np
import pytest

from conftest import pkg
from test_gpu_whole_body_frame import _model, _stick_figures

pytestmark = pytest.mark.gpu

H, W = 480, 640


def _detectors():
    PD = pkg("pose_detector")
    model = pkg("models.CocoPoseNet").CocoPoseNet()
    model.load_npz(pkg("synthetic").he_weights(0))
    return (PD.PoseDetector(model=model, device=0), pkg("face_detector").FaceDetector(model=_model("face"), device=0),
            pkg("hand_detector").HandDetector(model=_model("hand"), device=0))


@pytest.fixture(scope="module")
def dets():
    return _detectors()


@pytest.fixture
def eq_dets():
    """detectors whose every chain shape (pose at batch 1 and 4, FaceNet / HandNet chunks of 1, 2, 4, 8 and 16) is
    built with OPB_SMALL_BATCH=0: the variable is read when a chain is built.  Per test, so that their crop-map
    workspace (tens of GB for the hundreds of large crops of a random-weight frame) is freed before the next detectors
    grow theirs; the equal-tile tests come first in this module for the same reason."""
    with pytest.MonkeyPatch.context() as mp:
        mp.setenv("OPB_SMALL_BATCH", "0")
        d = _detectors()
        pose, face, hand = d
        frames = np.stack([pkg("synthetic").procedural_image(H, W, seed=s) for s in range(4)])
        pose.detect_batch(frames[:1])
        pose.detect_batch(frames)
        for k in (1, 2, 3, 5, 16):
            boxes = [(10 * i, 20, 10 * i + 60, 90) for i in range(k)]
            face.detect_crops(frames[0], boxes)
            hand.detect_crops(frames[0], boxes, ["left"] * k)
    return d


def _expected_parts(pose_det, poses):
    """test_gpu_whole_body_frame._expected_parts (the demo's boxes in its order under the skipping policy) without
    cutting the crops: PoseDetector.crop_image cannot cut a box that lies wholly below or right of the frame, and the
    boxes of random-weight persons can"""
    det = object.__new__(type(pose_det))
    det.engine = pose_det.engine
    det.crop_image = lambda img, bbox: None
    out = []
    for i, pose in enumerate(np.asarray(poses).reshape(-1, 18, 3)):
        pose = pose.copy()
        with np.errstate(all="ignore"):
            u = det.get_unit_length(pose)
        if not np.isfinite(u):
            continue
        _, fb = det.crop_face(None, pose, u)
        hands = det.crop_hands(None, pose, u)
        for side, bb in (("face", fb), ("left", hands["left"] and hands["left"]["bbox"]),
                         ("right", hands["right"] and hands["right"]["bbox"])):
            if bb is not None and bb[2] > bb[0] and bb[3] > bb[1]:
                out.append((i, side, tuple(int(v) for v in bb)))
    return out


def _launches(ds):
    return [d.engine.launch_count() for d in ds]


def _same_frame(a, b):
    """two (poses, scores, parts, owners, picture) tuples are equal bit for bit (float32 keypoint bytes included)"""
    assert np.array_equal(a[0], b[0]) and np.asarray(a[0]).shape == np.asarray(b[0]).shape
    assert np.array_equal(a[1], b[1])
    assert a[3] == b[3]
    assert [(k, bb) for k, bb, _ in a[2]] == [(k, bb) for k, bb, _ in b[2]]
    for (_, _, ka), (_, _, kb) in zip(a[2], b[2]):
        assert [p is None for p in ka] == [p is None for p in kb]
        for p, q in zip(ka, kb):
            if p is not None:
                assert p[0] == q[0] and p[1] == q[1]
                assert np.float32(p[2]).tobytes() == np.float32(q[2]).tobytes()
    if a[4] is None or b[4] is None:
        assert a[4] is None and b[4] is None
    else:
        assert np.array_equal(a[4], b[4]), "%d pixels differ" % int((a[4] != b[4]).any(2).sum())


def test_equal_tiles_noise_frames(eq_dets):
    pose, face, hand = eq_dets
    wb = pkg("whole_body")
    frames = [pkg("synthetic").procedural_image(H, W, seed=s) for s in (3, 4, 5, 6)]
    got = wb.detect_whole_body_batch(frames, pose, face, hand)
    assert len(got) == 4
    for f, frame in enumerate(frames):
        _same_frame(got[f], wb.detect_whole_body(frame, pose, face, hand))
    assert sum(len(g[2]) for g in got) > 0


def test_equal_tiles_injected_batch(eq_dets):
    """0 (zero maps), 1, 4 and 16 stick figures in one call"""
    import torch
    pose, face, hand = eq_dets
    wb = pkg("whole_body")
    frames = np.stack([pkg("synthetic").procedural_image(H, W, seed=20 + i) for i in range(4)])
    pafs, heats = [], []
    for i, n_person in enumerate((0, 1, 4, 16)):
        if n_person == 0:
            pafs.append(torch.zeros((1, 38, 46, 62), dtype=torch.float32, device="cuda"))
            heats.append(torch.zeros((1, 19, 46, 62), dtype=torch.float32, device="cuda"))
        else:
            (d_paf, d_heat), _, _ = _stick_figures(pose, frames[i], n_person, seed=i)
            pafs.append(d_paf)
            heats.append(d_heat)
    d_paf, d_heat = torch.cat(pafs).contiguous(), torch.cat(heats).contiguous()
    torch.cuda.synchronize()
    got = wb._detect_whole_body_batch(frames, pose, face, hand, True, d_paf.data_ptr(), d_heat.data_ptr())
    for f in range(4):
        one = wb._detect_whole_body(frames[f], pose, face, hand, True, pafs[f].data_ptr(), heats[f].data_ptr())
        _same_frame(got[f], one)
    assert len(got[0][0]) == 0 and got[0][2] == [] and np.array_equal(got[0][4], frames[0])
    assert all(len(got[f][2]) > 0 for f in (1, 2, 3))


@pytest.mark.parametrize("case", ["seed3", "seed5", "figures1", "figures16"])
def test_n1_equals_detect_whole_body(dets, case):
    pose, face, hand = dets
    wb = pkg("whole_body")
    if case.startswith("seed"):
        frame = pkg("synthetic").procedural_image(H, W, seed=int(case[4:]))
        inj = (None, None)
    else:
        frame = pkg("synthetic").procedural_image(H, W, seed=11)
        (d_paf, d_heat), _, _ = _stick_figures(pose, frame, int(case[7:]))
        inj = (d_paf.data_ptr(), d_heat.data_ptr())
    wb._detect_whole_body(frame, pose, face, hand, True, *inj)            # every chain shape built
    l0 = _launches(dets)
    one = wb._detect_whole_body(frame, pose, face, hand, True, *inj)
    l1 = _launches(dets)
    got = wb._detect_whole_body_batch(frame[None], pose, face, hand, True, *inj)
    l2 = _launches(dets)
    assert len(got) == 1
    _same_frame(got[0], one)
    assert [b - a for a, b in zip(l0, l1)] == [b - a for a, b in zip(l1, l2)]
    assert len(one[0]) and len(one[2])


def test_default_policy_batch_of_8(dets):
    pose, face, hand = dets
    wb = pkg("whole_body")
    frames = np.stack([pkg("synthetic").procedural_image(H, W, seed=30 + i) for i in range(8)])
    got = wb.detect_whole_body_batch(frames, pose, face, hand)
    ref = pose.detect_batch(frames)
    differ = total = 0
    for f in range(8):
        poses, scores = ref[f]
        g = got[f]
        assert np.array_equal(g[0], poses) and np.asarray(g[0]).shape == np.asarray(poses).shape
        assert np.array_equal(g[1], scores)
        exp = _expected_parts(pose, poses)
        assert [(o[0], o[1], p[1]) for o, p in zip(g[3], g[2])] == exp
        assert all(type(v) is int for _, b, _ in g[2] for v in b)
        assert np.array_equal(g[4], wb.draw_whole_body(frames[f], poses, g[2]))
        faces = [b for _, s, b in exp if s == "face"]
        hands = [(b, s) for _, s, b in exp if s != "face"]
        fk = iter(face.detect_crops(frames[f], faces) if faces else [])
        hk = iter(hand.detect_crops(frames[f], [b for b, _ in hands], [s for _, s in hands]) if hands else [])
        want = [next(fk) if s == "face" else next(hk) for _, s, _ in exp]
        differ += sum(a[2] != b for a, b in zip(g[2], want))
        total += len(exp)
    print("batch of 8: %d parts, %d keypoint lists differ from per-frame detect_crops" % (total, differ))
    assert total > 0


def _crop_launches(det, frames, results, kind):
    """launches of one detect_crops call with every face (or hand) crop of the batch"""
    boxes, types = [], []
    for g in results:
        for (k, b, _), (_, s) in zip(g[2], g[3]):
            if (k == "face") == (kind == "face"):
                boxes.append(b)
                types.append(s)
    if not boxes:
        return 0
    l0 = det.engine.launch_count()
    if kind == "face":
        det.detect_crops(frames[0], boxes)
    else:
        det.detect_crops(frames[0], boxes, types)
    return det.engine.launch_count() - l0


def _injected(pose, frames, n_person):
    """device maps [N,38|19,46,62] of n_person stick figures per frame (a different seed per frame)"""
    import torch
    params = pkg("entity").params
    in_w, in_h = pose.compute_optimal_size(frames[0], params["inference_img_size"])
    maps = [pkg("synthetic").eight_person_lowres(h=in_h // 8, w=in_w // 8, n_person=n_person, seed=f)
            for f in range(len(frames))]
    d_paf = torch.from_numpy(np.ascontiguousarray(np.stack([m[0] for m in maps]))).cuda()
    d_heat = torch.from_numpy(np.ascontiguousarray(np.stack([m[1] for m in maps]))).cuda()
    torch.cuda.synchronize()
    return d_paf, d_heat, (in_h, in_w)


def test_launch_count(dets):
    """pose: the batch resize + the launches of Engine.detect_batch at batch N on the same maps + 1 box launch + the
    picture (records -> poses, raster, paint); face / hand: one detect_crops call with all the batch's crops"""
    pose, face, hand = dets
    wb = pkg("whole_body")
    params = pkg("entity").params
    per_n = {}
    for n in (2, 8):
        frames = np.stack([pkg("synthetic").procedural_image(H, W, seed=30 + i) for i in range(n)])
        d_paf, d_heat, (in_h, in_w) = _injected(pose, frames, 4)
        map_w, map_h = pose.compute_optimal_size(frames[0], params["heatmap_size"])
        inj = (d_paf.data_ptr(), d_heat.data_ptr())
        wb._detect_whole_body_batch(frames, pose, face, hand, True, *inj)          # every chain shape built
        eng = pose.engine
        l0 = eng.launch_count()
        resized = eng.resize_linear_u8(frames, in_h, in_w)
        eng.detect_batch(resized, map_h, map_w, img_len=map_w, inject_paf=inj[0], inject_heat=inj[1])
        n_pose = eng.launch_count() - l0
        before = _launches(dets)
        got = wb._detect_whole_body_batch(frames, pose, face, hand, True, *inj)
        d = [b - a for a, b in zip(before, _launches(dets))]
        n_face = _crop_launches(face, frames, got, "face")
        n_hand = _crop_launches(hand, frames, got, "hand")
        assert n_face and n_hand
        n_draw = 3                                                                  # persons and parts in every frame
        assert d == [n_pose + 1 + n_draw, n_face, n_hand], (d, n_pose, n_face, n_hand)
        per_n[n] = d[0] - n_pose - 1
        before = _launches(dets)
        nodraw = wb._detect_whole_body_batch(frames, pose, face, hand, False, *inj)
        assert [b - a for a, b in zip(before, _launches(dets))] == [n_pose + 1, n_face, n_hand]
        for a, b in zip(nodraw, got):
            assert b[4] is not None
            _same_frame(a, b[:4] + (None,))
    assert per_n[2] == per_n[8] == 3                                                # picture launches do not grow with N


def test_errors_launch_nothing(dets):
    pose, face, hand = dets
    native, wb = pkg("_native"), pkg("whole_body")
    frames = np.stack([pkg("synthetic").procedural_image(H, W, seed=s) for s in (3, 4)])

    def nothing_launched(fn, exc):
        before = _launches(dets)
        with pytest.raises(exc):
            fn()
        assert _launches(dets) == before

    before = _launches(dets)
    assert wb.detect_whole_body_batch([], pose, face, hand) == []
    assert wb.detect_whole_body_batch(np.zeros((0, H, W, 3), np.uint8), pose, face, hand) == []
    assert _launches(dets) == before
    nothing_launched(lambda: wb.detect_whole_body_batch([frames[0], frames[1][:, :320]], pose, face, hand), ValueError)
    nothing_launched(lambda: wb.detect_whole_body_batch(frames.astype(np.float32), pose, face, hand), ValueError)
    nothing_launched(lambda: wb.detect_whole_body_batch(frames[..., 0], pose, face, hand), ValueError)
    nothing_launched(lambda: wb.detect_whole_body_batch(frames[0], pose, face, hand), ValueError)
    nothing_launched(lambda: wb.detect_whole_body_batch([frames[0][..., :2]], pose, face, hand), ValueError)
    nothing_launched(lambda: wb.detect_whole_body_batch(frames, pose, hand, face), ValueError)       # swapped slots
    nothing_launched(lambda: wb.detect_whole_body_batch(frames, face, pose, hand), ValueError)
    pose.precise = True
    try:
        nothing_launched(lambda: wb.detect_whole_body_batch(frames, pose, face, hand), ValueError)
    finally:
        pose.precise = False
    face.engine.device = 1                 # a detector on another device (checked before any device work)
    try:
        nothing_launched(lambda: wb.detect_whole_body_batch(frames, pose, face, hand), ValueError)
    finally:
        face.engine.device = 0
    pe = pose.engine
    # the C entry refuses the same, and bad sizes, before anything is enqueued
    for args in ((hand.engine, face.engine, frames, 368, 496, 320, 432), (face.engine, hand.engine, frames, 368, 490, 320, 432),
                 (face.engine, hand.engine, frames, 368, 496, 0, 432)):
        nothing_launched(lambda: pe.whole_body_batch(*args, 432, 368, 0.1, 368, 0.1), native.OpbError)
    nothing_launched(lambda: pe.whole_body_batch(face.engine, hand.engine, frames, 368, 496, 320, 432, 432, 36, 0.1, 368,
                                                 0.1), native.OpbError)
    nothing_launched(lambda: face.engine.whole_body_batch(face.engine, hand.engine, frames, 368, 496, 320, 432, 432, 368,
                                                          0.1, 368, 0.1), native.OpbError)
    # n < 1 at the C entry
    k = native.C.c_int(0)
    fp = np.zeros(1, np.int32)
    before = _launches(dets)
    rc = pe.lib.opb_whole_body_batch(pe.ctx, face.engine.ctx, hand.engine.ctx, native._ptr(frames), native.OPB_HOST, 0,
                                     H, W, 368, 496, 320, 432, 432.0, None, None, 368, 0.1, 368, 0.1,
                                     native._ptr(np.zeros(1, native.HEADER_DTYPE)),
                                     native._ptr(np.zeros(1, native.PERSON_DTYPE)), None, 0, native.C.byref(k),
                                     native._ptr(fp), None, None, None, None, None)
    assert rc == native.ERR_ARG and _launches(dets) == before


def test_record_status_raises_as_detect_batch(dets):
    """a result status (here: more persons than max_persons) raises what detect_batch raises for that frame"""
    _, face, hand = dets
    PD = pkg("pose_detector")
    model = pkg("models.CocoPoseNet").CocoPoseNet()
    model.load_npz(pkg("synthetic").he_weights(0))
    small = PD.PoseDetector(model=model, device=0, max_persons=1)
    frames = np.stack([pkg("synthetic").procedural_image(H, W, seed=s) for s in (3, 5)])
    with pytest.raises(Exception) as e_batch:
        small.detect_batch(frames)
    with pytest.raises(type(e_batch.value)) as e_wb:
        pkg("whole_body").detect_whole_body_batch(frames, small, face, hand)
    assert type(e_wb.value) is type(e_batch.value)
    print("status error:", e_batch.value, "|", e_wb.value)
