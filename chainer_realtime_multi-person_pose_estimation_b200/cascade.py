"""Haar cascade face detection on the device: a drop-in for `cv2.CascadeClassifier(...).detectMultiScale`.

    cascade = CascadeClassifier(cv2.data.haarcascades + "haarcascade_frontalface_alt.xml", engine)
    rects = cascade.detectMultiScale(gray_or_bgr, scaleFactor=1.2, minNeighbors=3, minSize=(1, 1))

Returns exactly the rectangles cv2 4.x returns (DESIGN.md, "Haar cascade"), as an int32 [n, 4] array of (x, y, w, h)
sorted by (y, x, w, h) -- cv2's own order changes from run to run -- or `()` when nothing is found, as cv2 does.

Supported cascades: the OpenCV XML format (`opencv-cascade-classifier`) with stageType BOOST, featureType HAAR, stumps
only and no tilted features (frontalface_alt / _default / _alt_tree, eye, frontalcatface, ...).  Trees with more than one
split (frontalface_alt2, eye_tree_eyeglasses), tilted features (frontalcatface_extended), LBP cascades and the old
`opencv-haar-classifier` format are refused with a ValueError naming the reason, rather than evaluated differently."""
import xml.etree.ElementTree as ET

import numpy as np


class HaarCascade(object):
    """Flat tables of one stump-based HAAR cascade, as opb_cascade_load takes them.

    window (w, h); stage_ntrees int32 [S]; stage_threshold float32 [S] (as stored, before OpenCV's 1e-5 margin);
    stump_feature int32 [T], stump_threshold / stump_left / stump_right float32 [T] (stage by stage);
    rects int32 [F, 3, 4] (x, y, w, h) and weights float32 [F, 3] (a third rect of weight 0 is absent)."""

    def __init__(self, window, stage_ntrees, stage_threshold, stump_feature, stump_threshold, stump_left, stump_right,
                 rects, weights):
        self.window = window
        self.stage_ntrees = stage_ntrees
        self.stage_threshold = stage_threshold
        self.stump_feature = stump_feature
        self.stump_threshold = stump_threshold
        self.stump_left = stump_left
        self.stump_right = stump_right
        self.rects = rects
        self.weights = weights


def _floats(text):
    return [float(v) for v in text.split()]


def load_haar_cascade(filename):
    """Parse an OpenCV cascade XML file into a HaarCascade.  ValueError for a cascade this package cannot evaluate
    exactly as cv2 does."""
    root = ET.parse(filename).getroot()
    node = root.find("cascade")
    if node is None:
        if len(root) and root[0].get("type_id") == "opencv-haar-classifier":
            raise ValueError("%s: old-format (opencv-haar-classifier) cascade is not supported" % filename)
        raise ValueError("%s: no <cascade> node: not an OpenCV cascade file" % filename)
    stage_type = (node.findtext("stageType") or "").strip()
    feature_type = (node.findtext("featureType") or "").strip()
    if stage_type != "BOOST":
        raise ValueError("%s: stageType %r is not supported (BOOST only)" % (filename, stage_type))
    if feature_type != "HAAR":
        raise ValueError("%s: featureType %r is not supported (HAAR only)" % (filename, feature_type))
    window = (int(node.findtext("width")), int(node.findtext("height")))
    ntrees, sthr, sfeat, sthr_t, sleft, sright = [], [], [], [], [], []
    for stage in node.find("stages"):
        if stage.find("parent") is not None or stage.find("next") is not None:
            raise ValueError("%s: stage trees are not supported" % filename)
        weak = stage.find("weakClassifiers")
        ntrees.append(len(weak))
        sthr.append(float(stage.findtext("stageThreshold")))
        for tree in weak:
            nodes = _floats(tree.findtext("internalNodes"))
            leaves = _floats(tree.findtext("leafValues"))
            if len(nodes) != 4 or len(leaves) != 2:
                raise ValueError("%s: trees with more than one split (or categorical splits) are not supported; "
                                 "stumps only" % filename)
            sfeat.append(int(nodes[2]))
            sthr_t.append(nodes[3])
            sleft.append(leaves[0])
            sright.append(leaves[1])
    features = list(node.find("features"))
    rects = np.zeros((len(features), 3, 4), np.int32)
    weights = np.zeros((len(features), 3), np.float32)
    for i, f in enumerate(features):
        if int((f.findtext("tilted") or "0").strip()):
            raise ValueError("%s: tilted features are not supported" % filename)
        rs = list(f.find("rects"))
        if not 1 <= len(rs) <= 3:
            raise ValueError("%s: feature %d has %d rects (1 to 3 supported)" % (filename, i, len(rs)))
        for j, r in enumerate(rs):
            v = r.text.split()
            rects[i, j] = [int(t) for t in v[:4]]
            weights[i, j] = np.float32(float(v[4]))
    sfeat = np.array(sfeat, np.int32)
    if len(sfeat) and (sfeat.min() < 0 or sfeat.max() >= len(features)):
        raise ValueError("%s: a stump names a feature that does not exist" % filename)
    return HaarCascade(window, np.array(ntrees, np.int32), np.array(sthr, np.float32), sfeat,
                       np.array(sthr_t, np.float32), np.array(sleft, np.float32), np.array(sright, np.float32),
                       rects, weights)


class CascadeClassifier(object):
    """cv2.CascadeClassifier(filename) evaluated on the device of `engine` (any detector's `.engine`, or a fresh context
    on GPU 0 when None).  A context holds one cascade at a time; each classifier reloads its tables when another one
    was loaded into the same context since its last call."""

    def __init__(self, filename, engine=None):
        try:
            from . import _native
            from .entity import params
            from .pose_detector import make_opb_params
        except ImportError:  # flat import, like the reference
            import _native
            from entity import params
            from pose_detector import make_opb_params
        self.tables = load_haar_cascade(filename)
        self.engine = engine if engine is not None else _native.Engine(0, make_opb_params(params))
        self.ensure_loaded()

    def ensure_loaded(self):
        if getattr(self.engine, "cascade_tables", None) is not self.tables:
            self.engine.cascade_load(self.tables)

    def detectMultiScale(self, image, scaleFactor=1.1, minNeighbors=3, minSize=(0, 0), maxSize=(0, 0)):
        """cv2's detectMultiScale: int32 [n, 4] (x, y, w, h) sorted by (y, x, w, h), or () when nothing is found.
        `image`: uint8 [H, W] gray or [H, W, 3] BGR (converted as cv2.cvtColor(image, COLOR_BGR2GRAY))."""
        self.ensure_loaded()
        rects = self.engine.cascade_detect(image, scaleFactor, minNeighbors, minSize, maxSize)
        return rects if len(rects) else ()
