"""The whole-body result picture of the reference's demo.py (:28-57) in one call, and the demo's whole frame in one call.

    res = draw_whole_body(img, poses, parts)                      # host: the cv2 calls demo.py makes
    res = draw_whole_body(img, poses, parts, engine=det.engine)   # device: the same pixels, one upload, one download
    poses, scores, parts, owners, res = detect_whole_body(img, pose_detector, face_detector, hand_detector)
    results = detect_whole_body_batch(frames, pose_detector, face_detector, hand_detector)   # one tuple per frame

`parts` lists (kind, bbox, keypoints) in drawing order -- demo.py's is, person by person, face, left hand, right hand:
kind "face" (70 keypoints) or "hand" (21), bbox (left, top, right, bottom) as PoseDetector.crop_face / crop_hands
return it, keypoints the list FaceDetector / HandDetector return from __call__ or detect_crops ([x, y, conf] or None,
in crop coordinates).  With `engine` (any detector's .engine) the picture is rasterised on the device by
opb_draw_whole_body, bit for bit the image of the host path (csrc/overlay.cuh)."""
import cv2
import numpy as np

try:
    from . import _native
    from .entity import params
    from .face_detector import draw_face_keypoints
    from .hand_detector import draw_hand_keypoints
    from .pose_detector import draw_person_pose
except ImportError:  # flat import, like the reference
    import _native
    from entity import params
    from face_detector import draw_face_keypoints
    from hand_detector import draw_hand_keypoints
    from pose_detector import draw_person_pose

_KINDS = {"face": _native.PART_FACE, "hand": _native.PART_HAND}


def _checked_parts(parts):
    """parts -> [(native kind, (l, t, r, b), keypoints)]; ValueError for an unknown kind, a keypoint count that does not
    match the kind, or a box that is not four int32 integers"""
    out = []
    lim = np.iinfo(np.int32)
    for i, part in enumerate(parts):
        try:
            kind, bbox, kps = part
        except (TypeError, ValueError):
            raise ValueError("part %d is not a (kind, bbox, keypoints) triple: %r" % (i, part))
        if not isinstance(kind, str) or kind not in _KINDS:
            raise ValueError("part %d: unknown kind %r (expected 'face' or 'hand')" % (i, kind))
        code = _KINDS[kind]
        if len(kps) != _native.PART_POINTS[code]:
            raise ValueError("part %d: a %s has %d keypoints, got %d" % (i, kind, _native.PART_POINTS[code], len(kps)))
        bbox = tuple(bbox)
        if len(bbox) != 4 or not all(isinstance(v, (int, np.integer)) and not isinstance(v, (bool, np.bool_))
                                     and lim.min <= v <= lim.max for v in bbox):
            raise ValueError("part %d: bbox must be four int32 integers (left, top, right, bottom): %r" % (i, bbox))
        out.append((code, bbox, kps))
    return out


def draw_whole_body(orig_img, poses, parts, engine=None):
    """cv2.addWeighted(orig_img, 0.6, draw_person_pose(orig_img, poses), 0.4, 0), then for every part its keypoints at
    (bbox[0], bbox[1]) (draw_face_keypoints / draw_hand_keypoints) and its box (cv2.rectangle, white, thickness 1).
    `poses` as PoseDetector.__call__ returns them (may be empty).  Returns a new image; orig_img is not modified.
    With `engine` the device draws the same pixels; it refuses (OpbError) a present joint outside the image or a
    coordinate of magnitude above 2^20."""
    checked = _checked_parts(parts)
    if engine is not None:
        return engine.draw_whole_body(orig_img, poses, checked)
    res = cv2.addWeighted(orig_img, 0.6, draw_person_pose(orig_img, poses), 0.4, 0)
    for code, bbox, kps in checked:
        draw = draw_face_keypoints if code == _native.PART_FACE else draw_hand_keypoints
        res = draw(res, kps, (bbox[0], bbox[1]))
        cv2.rectangle(res, (bbox[0], bbox[1]), (bbox[2], bbox[3]), (255, 255, 255), 1)
    return res


_SIDES = {_native.SIDE_FACE: "face", _native.SIDE_LEFT: "left", _native.SIDE_RIGHT: "right"}


def detect_whole_body(img, pose_detector, face_detector, hand_detector, draw=True):
    """demo.py's frame (:24-57) in one device call (opb_whole_body_frame): the pose pass, every person's crop_face and
    crop_hands boxes, FaceNet and HandNet on all crops (concurrently, on the face and the hand detector's contexts), and
    the result picture.  Returns (poses, scores, parts, owners, picture):
      poses, scores  exactly pose_detector(img).  The demo's own array ends with its hand joints moved by crop_hands'
                     in-place `+=`; that side effect is not reproduced.
      parts          the (kind, bbox, keypoints) list draw_whole_body takes, in the demo's order (per person: face,
                     left hand, right hand), bbox as Python ints, keypoints as the detectors return them.
      owners         (person index, "face" | "left" | "right") per part.
      picture        draw_whole_body(img, poses, parts), or None with draw=False.
    Unlike the demo, which raises on them, a person whose unit length is not finite (no limb of positive length) gets
    no part and a box of zero width or height is no part.  ValueError for a precise PoseDetector, detectors on
    different devices, or a face / hand detector in the wrong slot; a result status error raises as __call__ does.
    Afterwards pose_detector.draw_last_result(img) draws this frame's skeleton."""
    return _detect_whole_body(img, pose_detector, face_detector, hand_detector, draw)


def _checked_engines(pose_detector, face_detector, hand_detector):
    """(pose, face, hand) engines; ValueError for a precise PoseDetector, a detector in the wrong slot or detectors on
    different devices"""
    if getattr(pose_detector, "precise", False):
        raise ValueError("detect_whole_body runs the single-scale path; a precise PoseDetector is not supported")
    pe, fe, he = pose_detector.engine, face_detector.engine, hand_detector.engine
    if getattr(pe, "kp_channels", 0) != 0:
        raise ValueError("pose_detector must hold CocoPoseNet")
    if getattr(fe, "kp_channels", 0) != 71:
        raise ValueError("face_detector must hold FaceNet (71 output channels), got %d" % getattr(fe, "kp_channels", 0))
    if getattr(he, "kp_channels", 0) != 22:
        raise ValueError("hand_detector must hold HandNet (22 output channels), got %d" % getattr(he, "kp_channels", 0))
    if not pe.device == fe.device == he.device:
        raise ValueError("the detectors are on different devices (%d, %d, %d)" % (pe.device, fe.device, he.device))
    return pe, fe, he


def _frame_result(pose_detector, header, persons, table, faces, hands, picture, sx, sy):
    """one frame's (poses, scores, parts, owners, picture) from its records and its rows of the part table"""
    poses, scores = pose_detector._poses_from_records(header, persons, sx, sy)
    parts, owners = [], []
    for r in table:
        face = int(r["kind"]) == _native.PART_FACE
        kps = (faces if face else hands)[int(r["row"])]
        parts.append(("face" if face else "hand", (int(r["left"]), int(r["top"]), int(r["right"]), int(r["bottom"])), kps))
        owners.append((int(r["person"]), _SIDES[int(r["side"])]))
    return poses, scores, parts, owners, picture


def _detect_whole_body(img, pose_detector, face_detector, hand_detector, draw, inject_paf=None, inject_heat=None):
    """detect_whole_body with inject_paf / inject_heat: device maps [1,38,H/8,W/8] / [1,19,H/8,W/8] that replace the
    pose network's output, as in Engine.detect_batch (stick-figure persons for tests and benchmarks)"""
    pe, fe, he = _checked_engines(pose_detector, face_detector, hand_detector)
    img = np.asarray(img)
    if img.dtype != np.uint8 or img.ndim != 3 or img.shape[2] != 3:
        raise ValueError("img must be a uint8 [H, W, 3] BGR frame, got %s %s" % (img.dtype, img.shape))
    oh, ow = img.shape[:2]
    in_w, in_h = pose_detector.compute_optimal_size(img, params['inference_img_size'])
    map_w, map_h = pose_detector.compute_optimal_size(img, params['heatmap_size'])
    headers, persons, table, faces, hands, picture = pe.whole_body_frame(
        fe, he, img, in_h, in_w, map_h, map_w, map_w, params["face_inference_img_size"],
        params['face_heatmap_peak_thresh'], params["hand_inference_img_size"], params['hand_heatmap_peak_thresh'],
        draw=draw, inject_paf=inject_paf, inject_heat=inject_heat)
    pose_detector._last_scale = (ow / map_w, oh / map_h)
    return _frame_result(pose_detector, headers[0], persons[0], table, faces, hands, picture, ow / map_w, oh / map_h)


def detect_whole_body_batch(frames, pose_detector, face_detector, hand_detector, draw=True):
    """detect_whole_body for a batch of video frames in one device call (opb_whole_body_batch): all frames through one
    pose forward at batch N, one crop-box launch, the face crops of all frames through FaceNet and the hand crops
    through HandNet in shared chunks, and all pictures in one raster and one paint launch.
    `frames` is a uint8 [N, H, W, 3] array or a sequence of equally sized BGR frames.  Returns a list of N tuples
    (poses, scores, parts, owners, picture), each what detect_whole_body returns for that frame (with the pose pass at
    batch N: results equal detect_whole_body's bit for bit where the conv tiles are the same, see DESIGN 4.2); an empty
    batch returns [] and launches nothing.  ValueError, before anything is launched, for frames of different sizes, a
    wrong dtype or shape, and the detector errors of detect_whole_body; a frame's result status raises what
    PoseDetector.detect_batch raises for it.  Afterwards pose_detector.draw_last_result(frames[0]) draws the first
    frame's skeleton."""
    return _detect_whole_body_batch(frames, pose_detector, face_detector, hand_detector, draw)


def _checked_frames(frames):
    """frames -> contiguous uint8 [N, H, W, 3]; ValueError for a wrong dtype or shape or frames of different sizes"""
    if isinstance(frames, np.ndarray):
        batch = frames
        if batch.ndim != 4 or batch.shape[3] != 3 or batch.dtype != np.uint8:
            raise ValueError("frames must be a uint8 [N, H, W, 3] BGR batch, got %s %s" % (batch.dtype, batch.shape))
    else:
        items = [np.asarray(f) for f in frames]
        for i, f in enumerate(items):
            if f.dtype != np.uint8 or f.ndim != 3 or f.shape[2] != 3:
                raise ValueError("frame %d must be a uint8 [H, W, 3] BGR frame, got %s %s" % (i, f.dtype, f.shape))
            if f.shape != items[0].shape:
                raise ValueError("frame %d is %s, frame 0 is %s: a batch holds equally sized frames"
                                 % (i, f.shape, items[0].shape))
        if not items:
            return np.zeros((0, 0, 0, 3), np.uint8)
        batch = np.stack(items)
    if batch.shape[0] and (batch.shape[1] == 0 or batch.shape[2] == 0):
        raise ValueError("frames must not be empty images, got %s" % (batch.shape,))
    return np.ascontiguousarray(batch)


def _detect_whole_body_batch(frames, pose_detector, face_detector, hand_detector, draw, inject_paf=None,
                             inject_heat=None):
    """detect_whole_body_batch with inject_paf / inject_heat: device maps [N,38,H/8,W/8] / [N,19,H/8,W/8] that replace
    the pose network's output, as in Engine.detect_batch (stick-figure persons for tests and benchmarks)"""
    pe, fe, he = _checked_engines(pose_detector, face_detector, hand_detector)
    frames = _checked_frames(frames)
    if len(frames) == 0:
        return []
    oh, ow = frames.shape[1:3]
    in_w, in_h = pose_detector.compute_optimal_size(frames[0], params['inference_img_size'])
    map_w, map_h = pose_detector.compute_optimal_size(frames[0], params['heatmap_size'])
    headers, persons, table, frame_parts, faces, hands, pictures = pe.whole_body_batch(
        fe, he, frames, in_h, in_w, map_h, map_w, map_w, params["face_inference_img_size"],
        params['face_heatmap_peak_thresh'], params["hand_inference_img_size"], params['hand_heatmap_peak_thresh'],
        draw=draw, inject_paf=inject_paf, inject_heat=inject_heat)
    pose_detector._last_scale = (ow / map_w, oh / map_h)
    return [_frame_result(pose_detector, headers[f], persons[f], table[frame_parts[f]:frame_parts[f + 1]], faces, hands,
                          None if pictures is None else pictures[f], ow / map_w, oh / map_h)
            for f in range(len(frames))]
