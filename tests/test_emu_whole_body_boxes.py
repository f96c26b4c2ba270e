"""CPU (`-m "not gpu"`): the crop-box kernel of opb_whole_body_frame (csrc/whole_body.cuh) runs in the emulated library
(tests/cuda_emu) through the test hook opb_test_whole_body_boxes, in the non-contracting and the FMA-contracting build.
Unit lengths equal PoseDetector.get_unit_length bit for bit and boxes equal crop_face / crop_hands over several thousand
persons (tests/whole_body_cases.py): both unit-length branches with 8 or more terms, Pythagorean and near-integer edges,
negative edges near zero, persons without a positive limb and zero-width boxes."""
import ctypes as C
import os
import sys

import pytest

import whole_body_cases as W
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


def test_whole_body_boxes_emulated(emu_lib, monkeypatch):
    native = pkg("_native")
    monkeypatch.setattr(native, "_lib", emu_lib)
    engine = native.Engine(0, pkg("pose_detector").make_opb_params())
    total, stats = W.run_cases(engine)
    print("whole-body boxes: %d persons, %s" % (total, stats))
    assert total >= 5000
    W.check_out_of_range(engine)
    unit, boxes, present, parts = engine.test_whole_body_boxes(W._records(0), 1.0, 1.0)
    assert len(unit) == 0 and len(parts) == 0
