"""CPU (`-m "not gpu"`): opb_draw_whole_body -- the whole-body picture of demo.py:28-57 -- run under the CPU emulation
of tests/cuda_emu (see tests/test_emu_postprocess.py), with the test bodies of tests/test_gpu_draw_whole_body.py:
the device image must equal the host cv2 image bit for bit.

Every case runs against both emulated builds, -ffp-contract=off and the FMA-contracting one, so the blend of the paint
kernel is shown not to depend on the compiler's contraction choices.  Frames stay at 240 x 320 or below; the 640 x 480
demo flow, which needs the networks, runs on the GPU only."""
import ctypes as C
import os
import sys

import pytest

from conftest import pkg

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "cuda_emu"))
import build_emu  # noqa: E402
import test_gpu_draw_whole_body as G  # noqa: E402  (plain functions; the gpu mark belongs to that module only)


def _load(contract):
    native = pkg("_native")
    try:
        lib = C.CDLL(build_emu.build(contract=contract))
    except (RuntimeError, OSError) as e:     # no g++ / CUDA headers on this box: the harness, not the product, is missing
        pytest.skip("emulated build unavailable: %s" % str(e)[:200])
    for name, (res, args) in native._SIGNATURES.items():
        fn = getattr(lib, name)
        fn.restype = res
        fn.argtypes = args
    return lib


@pytest.fixture(scope="module", params=["nofma", "fma"])
def emu_lib(request):
    return _load(request.param == "fma")


@pytest.fixture()
def engine(emu_lib, monkeypatch):
    """For the duration of one test, Engine() binds the emulated library instead of libopb.so."""
    native = pkg("_native")
    monkeypatch.setattr(native, "_lib", emu_lib)
    return native.Engine(0, pkg("pose_detector").make_opb_params())


def test_random_frames_skeletons_and_parts(engine):
    G.test_random_frames_skeletons_and_parts(engine)


def test_segment_directions_and_clipping(engine):
    G.test_segment_directions_and_clipping(engine)


def test_overlapping_parts_overwrite_in_order(engine):
    G.test_overlapping_parts_overwrite_in_order(engine)


def test_blend_every_value_under_every_skeleton_colour(engine):
    G.test_blend_every_value_under_every_skeleton_colour(engine)


def test_empty_poses_and_parts(engine):
    G.test_empty_poses_and_parts(engine)


def test_errors_and_launch_count(engine):
    G.test_errors_and_launch_count(engine)
