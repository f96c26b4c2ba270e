"""ORACLE / TEST INFRASTRUCTURE ONLY.  Writes the cascade fixtures under tests/golden/:

    cascade_<name>_bgr.png, cascade_<name>_gray.png   the reference's data/<name>.png (person, dinner, people) as a BGR
                                                      frame and as cv2.cvtColor(BGR2GRAY) of it, lossless PNG
    cascade_outputs.npz                               cv2.CascadeClassifier.detectMultiScale's results on the gray
                                                      frames with haarcascade_frontalface_alt.xml, sorted by
                                                      (y, x, w, h) because cv2's own order changes from run to run

    python oracle/make_cascade_goldens.py

Needs the reference's data/ directory and cv2 (with cv2.data.haarcascades).  Keys of cascade_outputs.npz:
    <name>_<case>                            int32 [n, 4] (x, y, w, h) for every case of CASES
    <name>_raw_s1.2, <name>_raw_weights      the 1.2 / minSize (1, 1) raw candidates and their levelWeights (float64)
tests/haar_ref.py (cascade_fixtures) reads them back."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_DATA = os.environ.get("OPB_REFERENCE_DATA", "/root/reference/data")
NAMES = ("person", "dinner", "people")

# case key -> (scaleFactor, minNeighbors, minSize, maxSize)
CASES = {}
for _sf in (1.1, 1.2, 1.3):
    for _mn in (0, 1, 3, 5):
        CASES["mn%d_s%g" % (_mn, _sf)] = (_sf, _mn, (1, 1), (0, 0))
CASES["mn3_s1.2_min40"] = (1.2, 3, (40, 40), (0, 0))
CASES["mn0_s1.2_max60"] = (1.2, 0, (1, 1), (60, 60))
CASES["mn3_s1.2_min30_max100"] = (1.2, 3, (30, 30), (100, 100))
CASES["mn0_s1.1_min50x30"] = (1.1, 0, (50, 30), (0, 0))


def sort_rects(rects):
    rows = sorted((tuple(int(v) for v in r) for r in rects), key=lambda r: (r[1], r[0], r[2], r[3]))
    return np.array(rows, np.int32).reshape(-1, 4)


def main():
    import cv2
    cascade = cv2.CascadeClassifier(os.path.join(cv2.data.haarcascades, "haarcascade_frontalface_alt.xml"))
    gold = os.path.join(ROOT, "tests", "golden")
    out = {}
    for name in NAMES:
        bgr = cv2.imread(os.path.join(REF_DATA, name + ".png"), cv2.IMREAD_COLOR)
        gray = cv2.cvtColor(bgr, cv2.COLOR_BGR2GRAY)
        for kind, img in (("bgr", bgr), ("gray", gray)):
            path = os.path.join(gold, "cascade_%s_%s.png" % (name, kind))
            cv2.imwrite(path, img, [cv2.IMWRITE_PNG_COMPRESSION, 9])
            assert np.array_equal(cv2.imread(path, cv2.IMREAD_UNCHANGED), img)
            print("wrote", path, os.path.getsize(path), "bytes")
        for key, (sf, mn, mins, maxs) in CASES.items():
            out["%s_%s" % (name, key)] = sort_rects(cascade.detectMultiScale(gray, sf, mn, minSize=mins, maxSize=maxs))
        r, _, w = cascade.detectMultiScale3(gray, 1.2, 0, minSize=(1, 1), outputRejectLevels=True)
        pairs = sorted(((tuple(int(v) for v in a), float(b)) for a, b in zip(r, w)),
                       key=lambda p: (p[0][1], p[0][0], p[0][2], p[0][3]))
        out[name + "_raw_s1.2"] = np.array([p[0] for p in pairs], np.int32).reshape(-1, 4)
        out[name + "_raw_weights"] = np.array([p[1] for p in pairs], np.float64)
        print(name, bgr.shape, {k: len(out["%s_%s" % (name, k)]) for k in CASES})
    path = os.path.join(gold, "cascade_outputs.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    sys.exit(main())
