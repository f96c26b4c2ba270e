"""The whole-body result picture of the reference's demo.py (:28-57) in one call.

    res = draw_whole_body(img, poses, parts)                      # host: the cv2 calls demo.py makes
    res = draw_whole_body(img, poses, parts, engine=det.engine)   # device: the same pixels, one upload, one download

`parts` lists (kind, bbox, keypoints) in drawing order -- demo.py's is, person by person, face, left hand, right hand:
kind "face" (70 keypoints) or "hand" (21), bbox (left, top, right, bottom) as PoseDetector.crop_face / crop_hands
return it, keypoints the list FaceDetector / HandDetector return from __call__ or detect_crops ([x, y, conf] or None,
in crop coordinates).  With `engine` (any detector's .engine) the picture is rasterised on the device by
opb_draw_whole_body, bit for bit the image of the host path (csrc/overlay.cuh)."""
import cv2
import numpy as np

try:
    from . import _native
    from .face_detector import draw_face_keypoints
    from .hand_detector import draw_hand_keypoints
    from .pose_detector import draw_person_pose
except ImportError:  # flat import, like the reference
    import _native
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
