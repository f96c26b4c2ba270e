"""Cases and references of the face / hand crop pass run stage by stage (opb_test_keypoint_stages), shared by
tests/test_gpu_keypoint_stages.py and tests/test_emu_keypoint_stages.py.

The hook runs the launches of opb_keypoints_detect_crops on injected network-resolution maps instead of a network:
crop-resize into each chunk's canvases, the ragged align-corners upsample, the two smoothing passes and the arg-max.
Every stage is compared bit for bit with an independent reference applied to the reference of the stage before it:

  canvas     cv2.resize(flip?(canvas), (net, net)) and R.cv2_resize_linear_u8; the canvas is
             PoseDetector.crop_image, or crop_face's zero-padded square when vh < h or vw < w; padding slots are zero
  upsample   R.resize_bilinear_align_corners of the crop's [planes][net/8][net/8] maps to its own h x w
  axis 0     scipy.ndimage.gaussian_filter1d(axis=0), the first pass of gaussian_filter, stored as float32
  smoothed   scipy.ndimage.gaussian_filter(m, sigma=2.5) per plane (the reference's own call) and R.gaussian_smooth
  records    value = float32 max, count = len(np.where(g == g.max())[0]), key0 / key1 = the first two row-major tie
             positions of the mirrored map when flip is set
  keypoints  R.keypoints_from_heatmaps of the (mirrored) upsampled maps

and every word past the sizes the hook reports keeps the sentinel it was filled with."""
import cv2
import numpy as np
import scipy.ndimage as ndi

from conftest import pkg
from oracle import restate as R

NET = 368
H8 = NET // 8
FACE, HAND = 70, 21
THRESH = 0.1                                   # face_heatmap_peak_thresh == hand_heatmap_peak_thresh
TAIL = 4096
WORD = 0x7FA5A5A5                              # the hook's sentinel in float and record words
FH, FW, NF = 240, 320, 3                       # F = 3 frames of 240 x 320

# sizes (h, w) named in DESIGN.md 6: one pixel, the 46 x 46 identity, shrinking (< 46) and enlarging upsamples,
# 11 x 11 (the first size with only one reflection per border), 736 x 736 (exactly 2x down: cv2 takes INTER_AREA)
SMALL_SIZES = [(1, 1), (1, 40), (40, 1), (2, 3), (5, 7), (10, 10), (11, 11), (45, 46), (46, 46), (47, 47), (91, 92),
               (30, 520), (16, 16), (46, 16), (8, 32), (9, 65)]
LARGE_SIZES = [(367, 368), (368, 368), (369, 370), (401, 401), (1104, 300)]
TILE_SIZES = [(h, w) for h in (7, 8, 9) for w in (31, 32, 33, 64, 65)]      # around the 32 x 8 tile
PLACEMENTS = ("inside", "left", "top", "right", "bottom", "beyond_right", "beyond_bottom", "pad_h", "pad_w")
KINDS = 7


def chunk_slots(n):
    """kp_chunk_slots over a table of n crops: full chunks of 16, then the remainder rounded up to a power of two"""
    out = []
    while n > 0:
        s = 16 if n >= 16 else 1 << (n - 1).bit_length()
        out.append(s)
        n -= min(s, n)
    return out


def _place(rs, h, w, kind, flip, frame):
    """a crop row (left, top, right, bottom, flip, frame, vh, vw) of canvas h x w placed as `kind`"""
    vh, vw = h, w
    left = int(rs.randint(0, max(FW - w, 0) + 1))
    top = int(rs.randint(0, max(FH - h, 0) + 1))
    if kind == "left":
        left = -max(w // 2, 1)
    elif kind == "top":
        top = -max(h // 2, 1)
    elif kind == "right":
        left = FW - max(w // 2, 1)
    elif kind == "bottom":
        top = FH - max(h // 2, 1)
    elif kind == "beyond_right":
        left = FW + int(rs.randint(0, 9))
    elif kind == "beyond_bottom":
        top = FH + int(rs.randint(0, 9))
    elif kind in ("pad_h", "pad_w"):         # crop_face: an edge x edge square over a smaller extent inside the frame
        e = max(h, w, 2)
        h = w = vh = vw = e
        if kind == "pad_h":
            vh = int(rs.randint(1, e))
        else:
            vw = int(rs.randint(1, e))
        left, top = int(rs.randint(0, FW - vw + 1)), int(rs.randint(0, FH - vh + 1))
    return (left, top, left + w, top + h, int(flip), int(frame), vh, vw)


def _maps(rs, n, planes):
    """[n][planes + 1][46][46]; plane p of crop i is of kind (p + i) % 7, the background is 1e30"""
    m = np.zeros((n, planes + 1, H8, H8), np.float32)
    t = np.float32(THRESH)
    for i in range(n):
        for p in range(planes):
            k = (p + i) % KINDS
            a = m[i, p]
            if k == 0:                                        # Gaussian noise
                a[:] = rs.standard_normal((H8, H8))
            elif k == 1:                                      # constant: every pixel ties
                pass
            elif k == 2:                                      # two peaks at mirrored positions of one row
                a[15, 15] = a[15, 30] = 1.0
            elif k == 3:                                      # two peaks on different rows, not mirror images
                a[15, 15] = a[30, 30] = 1.0
            elif k == 4:                                      # at the float32 threshold, or one ulp above it
                a[:] = t if (i // KINDS) % 2 == 0 else np.nextafter(t, np.float32(1))
            elif k == 5:                                      # maxima on the last row and column
                a[:] = rs.standard_normal((H8, H8)) * np.float32(0.01)
                a[H8 - 1, H8 - 1] = 3.0
                a[H8 - 1, 7] = a[9, H8 - 1] = 2.5
            else:                                             # a steep step before the last row and column: the
                a[:] = rs.standard_normal((H8, H8))           # last output row / column must sample 45 exactly, or
                a[H8 - 2, :] = a[:, H8 - 2] = -1e10           # a 1e-14 weight on row / column 44 shows
        m[i, planes] = 1e30
    return m


def cases():
    """[(name, planes, frames [3][240][320][3], rows, maps)]: crop counts 1, 5, 16, 17, 21, 40 and 301"""
    rs = np.random.RandomState(2024)
    frames = rs.randint(0, 256, (NF, FH, FW, 3)).astype(np.uint8)
    calls = []

    def add(name, planes, rows):
        assert {r[5] for r in rows} == set(range(NF)) or len(rows) < NF
        calls.append((name, planes, frames, rows, _maps(rs, len(rows), planes)))

    # one crop: 736 x 736 around the frame (cut by all four borders), mirrored
    add("one", HAND, [(-200, -250, 536, 486, 1, 1, 736, 736)])
    # five crops (three padding slots of an 8-slot chunk): the large sizes, cut by the borders
    add("five", HAND, [_place(rs, h, w, PLACEMENTS[1 + i % 4], i % 2, i % NF) for i, (h, w) in enumerate(LARGE_SIZES)])
    # sixteen (one full chunk): the small sizes, every placement, both flips
    add("sixteen", FACE, [_place(rs, h, w, PLACEMENTS[i % len(PLACEMENTS)] if max(h, w) < FH else "inside", i % 2 == 1,
                                 i % NF) for i, (h, w) in enumerate(SMALL_SIZES)])
    # seventeen (16 + 1): widths and heights around the tile, plus two tie-preserving sizes
    rows = [_place(rs, h, w, PLACEMENTS[i % len(PLACEMENTS)], (i // 2) % 2, i % NF) for i, (h, w) in enumerate(TILE_SIZES)]
    rows += [_place(rs, 46, 46, "inside", 1, 0), _place(rs, 10, 10, "inside", 1, 2)]
    add("seventeen", FACE, rows)
    # twenty-one (16 + 5): every placement with and without flip, tie-preserving sizes among them
    sizes = [(46, 46), (16, 16), (10, 10), (23, 57), (60, 19), (12, 12), (33, 80), (46, 16), (2, 2)]
    rows = [_place(rs, *sizes[(i + f) % len(sizes)], kind, f, (2 * i + f) % NF)
            for i, kind in enumerate(PLACEMENTS) for f in (0, 1)]
    rows += [_place(rs, 46, 46, "inside", 1, 1), _place(rs, 9, 64, "inside", 0, 2), _place(rs, 46, 46, "pad_w", 1, 0)]
    add("twenty_one", HAND, rows)
    # forty (16 + 16 + 8): random sizes, placements, flips and frames
    rows = [_place(rs, int(rs.randint(1, 100)), int(rs.randint(1, 100)), PLACEMENTS[int(rs.randint(len(PLACEMENTS)))],
                   int(rs.randint(2)), i % NF) for i in range(40)]
    add("forty", FACE, rows)
    # about three hundred tiny crops: many tiles per launch for the binary search of the tile owner
    rows = [_place(rs, int(rs.randint(1, 25)), int(rs.randint(1, 25)), PLACEMENTS[int(rs.randint(len(PLACEMENTS)))],
                   int(rs.randint(2)), i % NF) for i in range(301)]
    add("tiny", HAND, rows)
    return calls


def source_canvas(frame, row):
    """the crop's canvas before the flip: crop_image, or the zero-padded square of crop_face"""
    left, top, right, bottom, flip, _, vh, vw = row
    h, w = bottom - top, right - left
    if vh == h and vw == w:
        if left >= frame.shape[1] or top >= frame.shape[0] or right <= 0 or bottom <= 0:
            return np.zeros((h, w, 3), np.uint8)     # crop_image's slices go negative here; its canvas is all zero
        return pkg("pose_detector").PoseDetector.crop_image(None, frame, (left, top, right, bottom))
    assert h == w and 0 <= left and 0 <= top and left + vw <= frame.shape[1] and top + vh <= frame.shape[0]
    face = frame[top:top + vh, left:left + vw]                  # face_detector.crop_face
    padded = np.zeros((h, w, 3), np.uint8)
    padded[0:face.shape[0], 0:face.shape[1]] = face
    return padded


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _word(x):
    return int(np.array(x, np.float32).view(np.uint32))


class Stats(object):
    def __init__(self):
        self.crops = self.canvas = self.up = self.tmp = self.smooth = self.records = 0
        self.pad_slots = self.pair_ties_flipped = self.at_thresh = self.above_thresh = self.all_tie = 0

    def __str__(self):
        return ("%d crops; %d canvas bytes, %d padding slots; %d upsampled, %d axis-0, %d smoothed floats; %d records "
                "(%d mirrored key pairs that differ from the unmirrored ones, %d maxima at the threshold, %d one ulp "
                "above, %d all-tie planes)" % (self.crops, self.canvas, self.pad_slots, self.up, self.tmp, self.smooth,
                                               self.records, self.pair_ties_flipped, self.at_thresh,
                                               self.above_thresh, self.all_tie))


def check_call(engine, call, stats):
    name, planes, frames, rows, maps = call
    n = len(rows)
    res = engine.test_keypoint_stages(frames, rows, NET, planes, maps, THRESH, tail=TAIL)
    slots = chunk_slots(n)
    hw = [(r[3] - r[1], r[2] - r[0]) for r in rows]
    floats = sum(planes * h * w for h, w in hw)
    assert res["sizes"] == (sum(slots) * NET * NET * 3, floats, n * planes), name

    # canvases, slot by slot; padding slots zero; nothing past the last slot
    canvas = res["canvas"]
    slot_px = NET * NET * 3
    first = s0 = 0
    for s in slots:
        nc = min(s, n - first)
        for j in range(s):
            got = canvas[(s0 + j) * slot_px:(s0 + j + 1) * slot_px].reshape(NET, NET, 3)
            if j >= nc:
                assert not got.any(), "%s: padding slot %d is not zero" % (name, s0 + j)
                stats.pad_slots += 1
                continue
            row = rows[first + j]
            src = source_canvas(frames[row[5]], row)
            if row[4]:
                src = cv2.flip(src, 1)
            src = np.ascontiguousarray(src)
            exp = cv2.resize(src, (NET, NET))
            assert np.array_equal(got, exp), "%s: canvas of crop %d %s differs from cv2.resize" % (name, first + j, row)
            assert np.array_equal(R.cv2_resize_linear_u8(src, (NET, NET)), exp)
        first += nc
        s0 += s
    assert (canvas[sum(slots) * slot_px:] == 0xA5).all(), "%s: a store past the last canvas slot" % name
    stats.canvas += sum(slots) * slot_px

    # ragged maps, crop by crop
    off = 0
    for i, (row, (h, w)) in enumerate(zip(rows, hw)):
        k = planes * h * w
        up = R.resize_bilinear_align_corners(maps[i:i + 1, :planes], (h, w))[0]
        assert up.dtype == np.float32
        got = res["up"][off:off + k].reshape(planes, h, w)
        bad = _bits(got) != _bits(up)
        assert not bad.any(), "%s: upsample of crop %d (%d x %d) differs at %d of %d floats, first at %s" % (
            name, i, h, w, bad.sum(), k, np.argwhere(bad)[0])
        ax0 = ndi.gaussian_filter1d(up, R.GAUSSIAN_SIGMA, axis=1, mode="reflect", truncate=4.0)
        assert ax0.dtype == np.float32
        got = res["tmp"][off:off + k].reshape(planes, h, w)
        bad = _bits(got) != _bits(ax0)
        assert not bad.any(), "%s: axis-0 pass of crop %d (%d x %d) differs at %d of %d floats, first at %s" % (
            name, i, h, w, bad.sum(), k, np.argwhere(bad)[0])
        g = np.stack([ndi.gaussian_filter(up[p], sigma=R.GAUSSIAN_SIGMA) for p in range(planes)])
        assert np.array_equal(_bits(g), _bits(R.gaussian_smooth(up)))
        got = res["smooth"][off:off + k].reshape(planes, h, w)
        bad = _bits(got) != _bits(g)
        assert not bad.any(), "%s: smoothed maps of crop %d (%d x %d) differ at %d of %d floats, first at %s" % (
            name, i, h, w, bad.sum(), k, np.argwhere(bad)[0])
        off += k

        flip = bool(row[4])
        for p in range(planes):
            m = g[p]
            mx = m.max()
            count = len(np.where(m == mx)[0])
            keys = np.flatnonzero((m[:, ::-1] if flip else m) == mx)[:2]
            rec = res["records"][i * planes + p]
            want = (_word(mx), count, int(keys[0]), int(keys[1]) if count >= 2 else -1)
            have = (_word(rec["value"]), int(rec["count"]), int(rec["key0"]), int(rec["key1"]))
            assert have == want, "%s: record of crop %d plane %d: %s, expected %s" % (name, i, p, have, want)
            if flip and count == 2 and keys[1] != np.flatnonzero(m == mx)[1]:
                stats.pair_ties_flipped += 1
            stats.at_thresh += int(mx == np.float32(THRESH))
            stats.above_thresh += int(mx == np.nextafter(np.float32(THRESH), np.float32(1)))
            stats.all_tie += int(count == h * w and h * w > 1)
        bg = np.full((1, h, w), 1e30, np.float32)
        ref = R.keypoints_from_heatmaps(np.concatenate([up[:, :, ::-1] if flip else up, bg]), THRESH)
        kps = res["keypoints"][i]
        for p, (a, b) in enumerate(zip(kps, ref)):
            assert (a is None) == (b is None), "%s: crop %d plane %d: %s vs %s" % (name, i, p, a, b)
            if a is not None:
                assert (a[0], a[1]) == (int(b[0]), int(b[1])) and _word(a[2]) == _word(b[2]), (name, i, p, a, b)
    assert off == floats
    for key in ("up", "tmp", "smooth"):
        assert (_bits(res[key][floats:]) == WORD).all(), "%s: a store past the ragged maps (%s)" % (name, key)
    assert (res["records"][n * planes:].view(np.uint32) == WORD).all(), "%s: a store past the records" % name
    stats.crops += n
    stats.up += floats
    stats.tmp += floats
    stats.smooth += floats
    stats.records += n * planes


def run_all(engine):
    stats = Stats()
    for call in cases():
        check_call(engine, call, stats)
    # the edge cases the maps were built for did occur
    assert stats.pad_slots >= 3 + 5 and stats.pair_ties_flipped > 0 and stats.at_thresh > 0
    assert stats.above_thresh > 0 and stats.all_tie > 0
    return stats


def check_argument_errors(engine):
    """bad crop rows, planes, net_size or frame index: OPB_ERR_ARG before anything is launched"""
    native = pkg("_native")
    frames = np.zeros((2, 20, 30, 3), np.uint8)
    good = (2, 3, 12, 9, 0, 1, 6, 10)
    maps = np.zeros((1, 3, H8, H8), np.float32)
    bad_rows = [(2, 3, 2, 9, 0, 0, 6, 0), (2, 9, 12, 3, 0, 0, 0, 10),            # empty canvas
                (2, 3, 12, 9, 2, 0, 6, 10),                                      # flip not 0 / 1
                (2, 3, 12, 9, 0, 2, 6, 10), (2, 3, 12, 9, 0, -1, 6, 10),         # frame index outside [0, 2)
                (2, 3, 12, 9, 0, 0, 7, 10), (2, 3, 12, 9, 0, 0, 6, 11),          # valid extent beyond the canvas
                (2, 3, 12, 9, 0, 0, -1, 10)]
    l0 = engine.launch_count()
    for row in bad_rows:
        try:
            engine.test_keypoint_stages(frames, [good, row], NET, 2, np.zeros((2, 3, H8, H8), np.float32), THRESH)
        except native.OpbError as e:
            assert "-2" in str(e), (row, e)
        else:
            raise AssertionError("row %s was accepted" % (row,))
    for net, planes in ((NET, 0), (NET, 1025), (360 + 4, 2), (8, 2), (0, 2)):
        try:
            engine.test_keypoint_stages(frames, [good], net, planes, maps, THRESH)
        except native.OpbError as e:
            assert "-2" in str(e), (net, planes, e)
        else:
            raise AssertionError("net_size %d, planes %d were accepted" % (net, planes))
    assert engine.launch_count() == l0
    res = engine.test_keypoint_stages(frames, [good], NET, 2, maps, THRESH)
    assert res["sizes"] == (NET * NET * 3, 2 * 6 * 10, 2) and engine.launch_count() == l0 + 5
