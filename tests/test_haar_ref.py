"""CPU: the NumPy restatement of detectMultiScale (tests/haar_ref.py) equals cv2 4.x, and the cascade loader refuses
what it cannot evaluate exactly.

Raw candidates (minNeighbors 0) are compared together with their final stage sums (detectMultiScale3's levelWeights),
which pins the float32 feature arithmetic and the double stage sums bit for bit.  Grouped results are compared for
minNeighbors 1, 3 and 5.  All comparisons are between lists sorted by (y, x, w, h): cv2's order varies between runs."""
import functools
import os

import numpy as np
import pytest

from conftest import pkg
import haar_ref as H

cv2 = pytest.importorskip("cv2")
HAAR_DIR = getattr(getattr(cv2, "data", None), "haarcascades", "")
if not os.path.isfile(os.path.join(HAAR_DIR, "haarcascade_frontalface_alt.xml")):
    pytest.skip("cv2.data.haarcascades has no haarcascade_frontalface_alt.xml", allow_module_level=True)


def xml(name):
    return os.path.join(HAAR_DIR, "haarcascade_%s.xml" % name)


@functools.lru_cache(None)
def tables(name):
    return pkg("cascade").load_haar_cascade(xml(name))


@functools.lru_cache(None)
def classifier(name):
    return cv2.CascadeClassifier(xml(name))


@functools.lru_cache(None)
def frames():
    return H.cascade_fixtures()


def cv_raw(name, gray, sf, min_size=(1, 1), max_size=(0, 0)):
    r, _, w = classifier(name).detectMultiScale3(gray, sf, 0, minSize=min_size, maxSize=max_size,
                                                 outputRejectLevels=True)
    return sorted((tuple(int(v) for v in a), float(b)) for a, b in zip(r, w))


def cv_grouped(name, gray, sf, mn, min_size=(1, 1), max_size=(0, 0)):
    return H.sort_rects(classifier(name).detectMultiScale(gray, sf, mn, minSize=min_size, maxSize=max_size))


def check(name, gray, sf, min_size=(1, 1), max_size=(0, 0), groups=(1, 3, 5)):
    raw = H.detect_raw(tables(name), gray, sf, min_size, max_size, with_weights=True)
    assert raw == cv_raw(name, gray, sf, min_size, max_size)
    for mn in groups:
        assert H.sort_rects(H.group_rectangles([r for r, _ in raw], mn)) == cv_grouped(name, gray, sf, mn, min_size,
                                                                                       max_size), mn
    return raw


def test_gray_conversion():
    f = frames()
    for n in ("person", "dinner", "people"):
        assert np.array_equal(H.bgr_to_gray(f[n + "_bgr"]), cv2.cvtColor(f[n + "_bgr"], cv2.COLOR_BGR2GRAY))
        assert np.array_equal(f[n + "_gray"], H.bgr_to_gray(f[n + "_bgr"]))


def test_resize_linear_exact():
    rng = np.random.default_rng(3)
    for _ in range(60):
        h, w = (int(v) for v in rng.integers(2, 300, 2))
        img = rng.integers(0, 256, (h, w), dtype=np.uint8)
        sc = np.float32(1.2 ** int(rng.integers(0, 12)))
        lh, lw = H.layer_size(h, w, sc)
        if lh < 1 or lw < 1:
            continue
        assert np.array_equal(H.resize_linear_exact(img, lw, lh),
                              cv2.resize(img, (lw, lh), interpolation=cv2.INTER_LINEAR_EXACT)), (h, w, sc)


@pytest.mark.parametrize("sf", [1.1, 1.2, 1.3])
@pytest.mark.parametrize("frame", ["person", "dinner", "people"])
def test_fixture_frames(frame, sf):
    raw = check("frontalface_alt", frames()[frame + "_gray"], sf)
    if sf == 1.2:
        assert len(raw) > 0


def test_recorded_outputs():
    """The recorded cv2 outputs the GPU tests also use equal the restatement."""
    mk = pytest.importorskip("oracle.make_cascade_goldens")
    f = frames()
    raw = functools.lru_cache(None)(
        lambda frame, sf, mins, maxs: H.detect_raw(tables("frontalface_alt"), f[frame + "_gray"], sf, mins, maxs))
    for frame in ("person", "people"):
        for key, (sf, mn, mins, maxs) in mk.CASES.items():
            if sf != 1.2:
                continue
            got = H.sort_rects(H.group_rectangles(raw(frame, sf, mins, maxs), mn))
            assert got == [tuple(r) for r in f["%s_%s" % (frame, key)].tolist()], (frame, key)


@pytest.mark.parametrize("min_size,max_size", [((30, 30), (0, 0)), ((1, 1), (60, 60)), ((40, 40), (100, 100)),
                                               ((50, 30), (0, 0)), ((0, 0), (45, 90))])
def test_min_max_size(min_size, max_size):
    check("frontalface_alt", frames()["person_gray"], 1.2, min_size, max_size)


@pytest.mark.parametrize("name", ["frontalface_default", "eye", "frontalface_alt_tree", "frontalcatface"])
def test_other_cascades(name):
    check(name, frames()["person_gray"], 1.2)


def test_odd_sizes_and_borders():
    """Odd frame sizes, and the face cut by each border of the frame."""
    g = frames()["person_gray"]
    faces = cv_grouped("frontalface_alt", g, 1.2, 3)
    assert len(faces) == 1
    x, y, w, h = faces[0]
    cx, cy = x + w // 2, y + h // 2
    crops = [g[:301, :457], g[37:, 11:], g[cy - 150:cy + 151, cx:cx + 255], g[cy - 150:cy + 151, cx - 255:cx],
             g[cy:cy + 203, cx - 160:cx + 161], g[cy - 203:cy, cx - 160:cx + 161]]
    for c in crops:
        check("frontalface_alt", np.ascontiguousarray(c), 1.2, groups=(1, 3))


def test_degenerate_frames():
    """A frame smaller than the window, exactly the window, and a flat frame give what cv2 gives (nothing)."""
    for shape in [(19, 40), (40, 19), (20, 20), (23, 21)]:
        g = np.random.default_rng(1).integers(0, 256, shape, dtype=np.uint8)
        check("frontalface_alt", g, 1.2, groups=(3,))
    raw = check("frontalface_alt", np.full((120, 160), 128, np.uint8), 1.1, groups=(3,))
    assert raw == []


@pytest.mark.parametrize("name,reason", [("frontalface_alt2", "more than one split"),
                                         ("eye_tree_eyeglasses", "more than one split"),
                                         ("frontalcatface_extended", "tilted")])
def test_loader_refuses(name, reason):
    with pytest.raises(ValueError, match=reason):
        pkg("cascade").load_haar_cascade(xml(name))


def test_loader_refuses_lbp_and_old_format(tmp_path):
    lbp = tmp_path / "lbp.xml"
    lbp.write_text('<?xml version="1.0"?><opencv_storage><cascade type_id="opencv-cascade-classifier">'
                   "<stageType>BOOST</stageType><featureType>LBP</featureType><height>24</height><width>24</width>"
                   "<stages></stages><features></features></cascade></opencv_storage>")
    with pytest.raises(ValueError, match="LBP"):
        pkg("cascade").load_haar_cascade(str(lbp))
    old = tmp_path / "old.xml"
    old.write_text('<?xml version="1.0"?><opencv_storage><haar type_id="opencv-haar-classifier"><size>20 20</size>'
                   "</haar></opencv_storage>")
    with pytest.raises(ValueError, match="old-format"):
        pkg("cascade").load_haar_cascade(str(old))


def test_loader_tables():
    t = tables("frontalface_alt")
    assert t.window == (20, 20)
    assert len(t.stage_ntrees) == 22 and int(t.stage_ntrees.sum()) == 2135 == len(t.stump_feature)
    assert t.stage_ntrees[:2].tolist() == [3, 16]
    r = t.rects
    assert (r[..., 0] >= 0).all() and (r[..., 0] + r[..., 2] <= 20).all() and (r[..., 1] + r[..., 3] <= 20).all()
