"""CPU (`-m "not gpu"`): conv1_1 through opb_test_conv_first of the emulated library (tests/cuda_emu), bit for bit
against the NumPy restatement in conv_first_ref.py, on one small frame with partial tiles in both directions, in
all three precisions and both input kinds, in the non-contracting and the FMA-contracting build."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

import conv_first_ref as R
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
def emu_native(emu_lib, monkeypatch):
    native = pkg("_native")
    monkeypatch.setattr(native, "_lib", emu_lib)
    monkeypatch.setenv("OPB_EMU_SMS", "1")   # one persistent block walks every tile
    return native


@pytest.mark.parametrize("kind", ["u8_255", "u8_256", "f32"])
def test_conv_first_emulated(emu_native, kind):
    n, h, w = 2, 11, 37                          # 2 x 2 tiles per image, both partial
    W, b = R.make_weights(7)
    if kind == "f32":
        x = R.make_frame_f32(8, n, h, w)
        acc = R.conv_first_acc(x, W, b)
        denom = 255.0
    else:
        denom = 255.0 if kind == "u8_255" else 256.0
        x = R.make_frame_u8(8, n, h, w)
        acc = R.conv_first_acc(R.preprocess_u8(x, denom), W, b)
    eng = emu_native.Engine(0, pkg("pose_detector").make_opb_params())
    for mode, prec in (("fast", emu_native.PRECISION_FAST), ("parity", emu_native.PRECISION_PARITY),
                       ("comp", emu_native.PRECISION_COMP)):
        got = eng.test_conv_first(x, W, b, prec, u8_denom=denom)
        assert np.array_equal(got, R.encode(acc, mode)), mode
