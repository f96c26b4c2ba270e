"""CPU (`-m "not gpu"`): the face / hand crop pass of opb_keypoints_detect_crops run stage by stage from injected maps
(opb_test_keypoint_stages, tests/keypoint_stages.py) in the emulated library (tests/cuda_emu), in the non-contracting
and the FMA-contracting build: crop-resize, ragged upsample, both smoothing passes and the arg-max of seven crop tables
(1 to 301 crops, 70 and 21 planes, three frames), every stored value bit for bit against cv2, scipy and the restated
reference, with sentinels past every buffer.  No network runs, so the whole set takes minutes, not hours."""
import ctypes as C
import os
import sys

import pytest

import keypoint_stages as K
from conftest import pkg

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "cuda_emu"))
import build_emu  # noqa: E402


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


@pytest.fixture()
def engine(emu_lib, monkeypatch):
    native = pkg("_native")
    monkeypatch.setattr(native, "_lib", emu_lib)
    return native.Engine(0, pkg("pose_detector").make_opb_params())


def test_keypoint_stages_emulated(engine):
    stats = K.run_all(engine)
    print("keypoint stages: %s" % stats)


def test_keypoint_stages_argument_errors_emulated(engine):
    K.check_argument_errors(engine)
