"""NumPy restatement of cv2.CascadeClassifier.detectMultiScale for stump-based HAAR cascades (OpenCV 4.x,
objdetect/cascadedetect.cpp and imgproc's INTER_LINEAR_EXACT resize), pinned against cv2 by
tests/test_haar_ref.py.  The device kernels of csrc/cascade.cuh are tested against it window by window.

Every float32 step below is one IEEE operation on float32 NumPy scalars or arrays, so no step is contracted."""
import os

import numpy as np

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
FIXTURES = ("person", "dinner", "people")
THRESHOLD_EPS = np.float32(1e-5)
GROUP_EPS = 0.2


def bgr_to_gray(img):
    """cv2.cvtColor(img, COLOR_BGR2GRAY) on uint8: (B*3735 + G*19235 + R*9798 + 2^14) >> 15."""
    a = img.astype(np.int32)
    return ((a[..., 0] * 3735 + a[..., 1] * 19235 + a[..., 2] * 9798 + (1 << 14)) >> 15).astype(np.uint8)


def linear_exact_axis(dst_n, src_n):
    """Source indices and 8-bit coefficients of one axis of resize(..., INTER_LINEAR_EXACT):
    f = (d + 0.5) * (1 / (dst/src)) - 0.5 in double, s = floor(f), c1 = rint((f - s) * 256), c0 = 256 - c1; both
    indices clamp to the source (a clamped pair reads one pixel with weight 256)."""
    scale = 1.0 / (dst_n / src_n)
    f = (np.arange(dst_n, dtype=np.float64) + 0.5) * scale - 0.5
    s = np.floor(f)
    c1 = np.rint((f - s) * 256).astype(np.int64)
    s = s.astype(np.int64)
    return np.clip(s, 0, src_n - 1), np.clip(s + 1, 0, src_n - 1), 256 - c1, c1


def resize_linear_exact(img, w, h):
    """cv2.resize(img, (w, h), interpolation=cv2.INTER_LINEAR_EXACT) on a uint8 gray image: horizontal sums in
    8.8 fixed point, vertical in 16.16, (v + 2^15) >> 16."""
    x0, x1, a0, a1 = linear_exact_axis(w, img.shape[1])
    y0, y1, b0, b1 = linear_exact_axis(h, img.shape[0])
    im = img.astype(np.int64)
    hr = im[:, x0] * a0 + im[:, x1] * a1
    v = hr[y0] * b0[:, None] + hr[y1] * b1[:, None]
    return ((v + (1 << 15)) >> 16).astype(np.uint8)


def integrals(img):
    """(sum, sqsum) as (h+1) x (w+1) uint32 with a zero first row and column; OpenCV's int32 sqsum wraps at 640x480,
    and only window differences are used, so uint32 arithmetic gives the same bits."""
    h, w = img.shape
    s = np.zeros((h + 1, w + 1), np.uint32)
    q = np.zeros((h + 1, w + 1), np.uint32)
    a = img.astype(np.uint32)
    s[1:, 1:] = a.cumsum(0, dtype=np.uint32).cumsum(1, dtype=np.uint32)
    q[1:, 1:] = (a * a).cumsum(0, dtype=np.uint32).cumsum(1, dtype=np.uint32)
    return s, q


def scales(h, w, window, min_size=(0, 0), max_size=(0, 0), scale_factor=1.1):
    """The float32 scale list of detectMultiScaleNoGrouping."""
    win_w, win_h = window
    max_w, max_h = max_size
    if max_w == 0 or max_h == 0:
        max_w, max_h = w, h
    out = []
    factor = 1.0
    while True:
        ww, wh = int(np.rint(win_w * factor)), int(np.rint(win_h * factor))
        if ww > max_w or wh > max_h or ww > w or wh > h:
            break
        if not (ww < min_size[0] or wh < min_size[1]):
            out.append(np.float32(factor))
        factor *= scale_factor
    return out


def layer_size(h, w, sc):
    """(h, w) of the pyramid layer of float32 scale sc: cvRound(size / sc) in float32."""
    return int(np.rint(np.float32(h) / sc)), int(np.rint(np.float32(w) / sc))


class Layer(object):
    def __init__(self, gray, sc):
        self.sc = sc
        self.h, self.w = layer_size(gray.shape[0], gray.shape[1], sc)
        self.img = resize_linear_exact(gray, self.w, self.h)
        self.sum, self.sqsum = integrals(self.img)
        self.ystep = 1 if sc >= 2 else 2


def _rect_sum(ii, ys, xs, r):
    x, y, w, h = (int(v) for v in r)
    y0, x0 = ys + y, xs + x
    return (ii[y0, x0] - ii[y0, x0 + w] - ii[y0 + h, x0] + ii[y0 + h, x0 + w]).astype(np.int32)


def eval_windows(cascade, layer, ys, xs):
    """Result code and final stage sum of the windows with top-left (ys[i], xs[i]) of one layer (runAt):
    -1 when the window's variance test fails, -k when stage k rejects it, 1 when it passes every stage."""
    win_w, win_h = cascade.window
    n = len(ys)
    code = np.ones(n, np.int32)
    wsum = np.zeros(n, np.float64)
    nr = (1, 1, win_w - 2, win_h - 2)
    area = float((win_w - 2) * (win_h - 2))
    valsum = _rect_sum(layer.sum, ys, xs, nr).astype(np.float64)
    valsq = (_rect_sum(layer.sqsum, ys, xs, nr).astype(np.int64) & 0xFFFFFFFF).astype(np.float64)
    nf = area * valsq - valsum * valsum
    vnf = np.ones(n, np.float32)
    pos = nf > 0
    vnf[pos] = (1.0 / np.sqrt(nf[pos])).astype(np.float32)
    ok = pos & (area * vnf.astype(np.float64) < 0.1)
    code[~ok] = -1
    live = np.nonzero(ok)[0]
    t0 = 0
    for k, (nt, st) in enumerate(zip(cascade.stage_ntrees, cascade.stage_threshold)):
        if not len(live):
            break
        thr = np.float32(st) - THRESHOLD_EPS
        ly, lx, lv = ys[live], xs[live], vnf[live]
        acc = np.zeros(len(live), np.float64)
        for t in range(t0, t0 + int(nt)):
            fi = cascade.stump_feature[t]
            r, wt = cascade.rects[fi], cascade.weights[fi]
            ret = (wt[0] * _rect_sum(layer.sum, ly, lx, r[0]).astype(np.float32)
                   + wt[1] * _rect_sum(layer.sum, ly, lx, r[1]).astype(np.float32))
            if wt[2] != 0:
                ret = ret + wt[2] * _rect_sum(layer.sum, ly, lx, r[2]).astype(np.float32)
            value = ret * lv
            leaf = np.where(value < cascade.stump_threshold[t], cascade.stump_left[t], cascade.stump_right[t])
            acc = acc + leaf.astype(np.float64)
        t0 += int(nt)
        wsum[live] = acc
        rej = acc < np.float64(thr)
        code[live[rej]] = -k
        live = live[~rej]
    return code, wsum


def pyramid(gray, window, scale_factor, min_size=(0, 0), max_size=(0, 0)):
    h, w = gray.shape
    return [Layer(gray, sc) for sc in scales(h, w, window, min_size, max_size, scale_factor)]


def layer_windows(cascade, layer):
    """Every window the scan can visit in one layer, before the skip rule: y and x over the working size in ystep."""
    win_w, win_h = cascade.window
    wh, ww = layer.h + 1 - win_h, layer.w + 1 - win_w
    ys, xs = np.meshgrid(np.arange(0, max(wh, 0), layer.ystep), np.arange(0, max(ww, 0), layer.ystep), indexing="ij")
    return ys.ravel(), xs.ravel()


def scan_layer(cascade, layer, code):
    """CascadeClassifierInvoker over one layer, given the codes of layer_windows: x restarts at 0 on every row, and a
    window rejected by stage 0 (code 0) makes the scan skip the next x.  Returns the visited passing (x, y)."""
    win_w, win_h = cascade.window
    wh, ww = layer.h + 1 - win_h, layer.w + 1 - win_w
    if wh <= 0 or ww <= 0:
        return []
    nx = len(range(0, ww, layer.ystep))
    grid = code.reshape(-1, nx)
    out = []
    for j, y in enumerate(range(0, wh, layer.ystep)):
        row = grid[j]
        i = 0
        while i < nx:
            c = row[i]
            if c > 0:
                out.append((i * layer.ystep, y))
            i += 2 if c == 0 else 1
    return out


def candidate_rect(cascade, layer, x, y, h, w):
    """Rect(cvRound(x*sc), cvRound(y*sc), cvRound(winW*sc), cvRound(winH*sc)) in float32, clipped to the h x w frame
    (cv2 4.13 returns rects that end past the frame cut at its edge)."""
    sc = layer.sc
    rx, ry = int(np.rint(np.float32(x) * sc)), int(np.rint(np.float32(y) * sc))
    rw, rh = int(np.rint(np.float32(cascade.window[0]) * sc)), int(np.rint(np.float32(cascade.window[1]) * sc))
    return (rx, ry, min(rx + rw, w) - rx, min(ry + rh, h) - ry)


def detect_raw(cascade, gray, scale_factor=1.1, min_size=(0, 0), max_size=(0, 0), with_weights=False):
    """detectMultiScale(..., minNeighbors=0) as a sorted list of (x, y, w, h); with_weights: (rect, final stage sum)
    pairs, the levelWeights of detectMultiScale3(..., outputRejectLevels=True)."""
    out = []
    for layer in pyramid(gray, cascade.window, scale_factor, min_size, max_size):
        ys, xs = layer_windows(cascade, layer)
        code, wsum = eval_windows(cascade, layer, ys, xs)
        nx = len(np.unique(xs)) if len(xs) else 0
        for x, y in scan_layer(cascade, layer, code):
            i = (y // layer.ystep) * nx + x // layer.ystep
            r = candidate_rect(cascade, layer, x, y, gray.shape[0], gray.shape[1])
            out.append((r, float(wsum[i])) if with_weights else r)
    return sorted(out)


def _similar(a, b, eps):
    delta = eps * (min(a[2], b[2]) + min(a[3], b[3])) * 0.5
    return (abs(a[0] - b[0]) <= delta and abs(a[1] - b[1]) <= delta
            and abs(a[0] + a[2] - b[0] - b[2]) <= delta and abs(a[1] + a[3] - b[1] - b[3]) <= delta)


def group_rectangles(rects, group_threshold, eps=GROUP_EPS):
    """cv2.groupRectangles(rects, group_threshold, eps) as detectMultiScale applies it, output sorted."""
    rects = [tuple(int(v) for v in r) for r in rects]
    if group_threshold <= 0 or not rects:
        return sorted(rects)
    n = len(rects)
    parent = list(range(n))

    def find(i):
        while parent[i] != i:
            parent[i] = parent[parent[i]]
            i = parent[i]
        return i

    for i in range(n):
        for j in range(i + 1, n):
            if _similar(rects[i], rects[j], eps):
                a, b = find(i), find(j)
                if a != b:
                    parent[b] = a
    roots = sorted({find(i) for i in range(n)})
    cls = {r: k for k, r in enumerate(roots)}
    sums = np.zeros((len(roots), 4), np.int64)
    cnt = np.zeros(len(roots), np.int64)
    for i, r in enumerate(rects):
        k = cls[find(i)]
        sums[k] += r
        cnt[k] += 1
    avg = []
    for k in range(len(roots)):
        s = np.float32(1.0) / np.float32(cnt[k])
        avg.append(tuple(int(np.rint(np.float32(v) * s)) for v in sums[k]))
    out = []
    for i, r1 in enumerate(avg):
        n1 = int(cnt[i])
        if n1 <= group_threshold:
            continue
        keep = True
        for j, r2 in enumerate(avg):
            n2 = int(cnt[j])
            if j == i or n2 <= group_threshold:
                continue
            dx, dy = int(np.rint(r2[2] * eps)), int(np.rint(r2[3] * eps))
            if (r1[0] >= r2[0] - dx and r1[1] >= r2[1] - dy and r1[0] + r1[2] <= r2[0] + r2[2] + dx
                    and r1[1] + r1[3] <= r2[1] + r2[3] + dy and (n2 > max(3, n1) or n1 < 3)):
                keep = False
                break
        if keep:
            out.append(r1)
    return sorted(out)


def detect_multi_scale(cascade, img, scale_factor=1.1, min_neighbors=3, min_size=(0, 0), max_size=(0, 0)):
    """cv2.CascadeClassifier.detectMultiScale on a gray [H,W] or BGR [H,W,3] uint8 image, sorted by (y, x, w, h)."""
    gray = bgr_to_gray(img) if img.ndim == 3 else img
    raw = detect_raw(cascade, gray, scale_factor, min_size, max_size)
    return sort_rects(group_rectangles(raw, min_neighbors))


def sort_rects(rects):
    """The canonical order of the device results: by (y, x, w, h)."""
    return sorted((tuple(int(v) for v in r) for r in rects), key=lambda r: (r[1], r[0], r[2], r[3]))


def cascade_fixtures():
    """The cascade fixtures of tests/golden (written by oracle/make_cascade_goldens.py) as one dict: <name>_bgr and
    <name>_gray uint8 frames (lossless PNG, decoded with cv2) and cv2's recorded outputs of cascade_outputs.npz."""
    import cv2
    out = {}
    for name in FIXTURES:
        for kind in ("bgr", "gray"):
            img = cv2.imread(os.path.join(GOLDEN, "cascade_%s_%s.png" % (name, kind)), cv2.IMREAD_UNCHANGED)
            if img is None:
                raise FileNotFoundError("tests/golden/cascade_%s_%s.png" % (name, kind))
            out["%s_%s" % (name, kind)] = img
    with np.load(os.path.join(GOLDEN, "cascade_outputs.npz")) as f:
        out.update({k: f[k] for k in f.files})
    return out
