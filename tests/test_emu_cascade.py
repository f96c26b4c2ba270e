"""CPU (`-m "not gpu"`): the cascade kernels of csrc/cascade.cuh run in the emulated library (tests/cuda_emu) on a small
crop around the face of the person fixture, gray and BGR: every window's result code and final stage sum equal the
NumPy restatement (tests/haar_ref.py) bit for bit, and detectMultiScale equals it, in the non-contracting and the
FMA-contracting build."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

import haar_ref as H
from conftest import pkg

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "cuda_emu"))
import build_emu  # noqa: E402

cv2 = pytest.importorskip("cv2")
XML = os.path.join(getattr(getattr(cv2, "data", None), "haarcascades", ""), "haarcascade_frontalface_alt.xml")
if not os.path.isfile(XML):
    pytest.skip("cv2.data.haarcascades has no haarcascade_frontalface_alt.xml", allow_module_level=True)


@pytest.fixture(scope="module", params=[False, True], ids=["nocontract", "contract"])
def emu_lib(request):
    native = pkg("_native")
    try:
        lib = C.CDLL(build_emu.build(contract=request.param))
    except (RuntimeError, OSError) as e:     # no g++ / CUDA headers on this box: the harness, not the product, is missing
        pytest.skip("emulated build unavailable: %s" % str(e)[:200])
    for name, (res, args) in native._SIGNATURES.items():
        fn = getattr(lib, name)
        fn.restype = res
        fn.argtypes = args
    return lib


def test_cascade_emulated(emu_lib, monkeypatch):
    native = pkg("_native")
    monkeypatch.setattr(native, "_lib", emu_lib)
    f = H.cascade_fixtures()
    bgr = np.ascontiguousarray(f["person_bgr"][30:131, 330:431])     # 101 x 101 around the face
    gray = H.bgr_to_gray(bgr)
    cc = pkg("cascade").CascadeClassifier(XML, native.Engine(0, pkg("pose_detector").make_opb_params()))
    ref_c, ref_s = [], []
    for layer in H.pyramid(gray, cc.tables.window, 1.2, (1, 1)):
        ys, xs = H.layer_windows(cc.tables, layer)
        c, s = H.eval_windows(cc.tables, layer, ys, xs)
        ref_c.append(c)
        ref_s.append(s)
    ref_c, ref_s = np.concatenate(ref_c), np.concatenate(ref_s)
    assert (ref_c == 1).any()
    for img in (gray, bgr):
        codes, sums = cc.engine.test_cascade_windows(img, 1.2, (1, 1))
        assert np.array_equal(codes, ref_c)
        assert np.array_equal(sums.view(np.int64), ref_s.view(np.int64))
        for mn in (0, 3):
            want = H.detect_multi_scale(cc.tables, gray, 1.2, mn, (1, 1))
            got = cc.detectMultiScale(img, 1.2, mn, (1, 1))
            assert [tuple(int(v) for v in r) for r in (got if len(got) else [])] == want, mn
