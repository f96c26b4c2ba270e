"""CPU (`-m "not gpu"`): the crop-box kernel of opb_whole_body_batch (csrc/whole_body.cuh, one block per frame) runs in
the emulated library (tests/cuda_emu) through the test hook opb_test_whole_body_boxes_batch, in the non-contracting and
the FMA-contracting build, on one batch that mixes frames of every family of tests/whole_body_cases.py, a frame with an
error status, a frame with persons but no peaks, an empty frame and a frame of more than 256 persons (the kernel's
chunk loop).  Each frame's section must equal whole_body_cases.reference for that frame alone, with its status
reported per frame."""
import ctypes as C
import os
import sys

import numpy as np
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


def _batch(rs):
    """[(n_peaks, n_persons, status, records)] of one batch, and the frames' sx = sy"""
    frames = [
        (1, 200, 0, W.random_persons(rs, 200)),
        (1, 180, 0, W.branch2_persons(rs, 180)),
        (1, 3, -4, W.random_persons(rs, 3)),               # an error status: nothing but the status
        (1, 150, 0, W.near_integer_persons(rs, 150)),
        (0, 5, 0, W.random_persons(rs, 5)),                # persons but no peaks: _poses_from_records gives none
        (1, 120, 0, W.small_persons(rs, 120)),
        (1, 0, 0, W.random_persons(rs, 0)),                # an empty frame
        (1, 90, 0, W.degenerate_persons(rs, 90)),
        (1, 300, 0, W.random_persons(rs, 300)),            # more than WB_THREADS persons: two chunks
    ]
    return frames


def _run(engine, frames, cap, s):
    native = pkg("_native")
    n = len(frames)
    headers = np.zeros(n, native.HEADER_DTYPE)
    persons = W._records(n * cap).reshape(n, cap)
    for f, (n_peaks, n_persons, status, rec) in enumerate(frames):
        headers[f] = (n_peaks, n_persons, status, 0)
        persons[f, :len(rec)] = rec
    return engine.test_whole_body_boxes_batch(headers, persons, s, s)


def _check_frame(engine, got, frame, s):
    n_peaks, n_persons, status, rec = frame
    assert got["status"] == status
    if status != 0 or n_peaks == 0 or n_persons == 0:
        assert len(got["parts"]) == 0 and len(got["face"]) == 0 and len(got["hand"]) == 0
        return 0
    r_unit, r_boxes, r_present, r_kept = W.reference(engine, rec, s, s)
    unit = got["unit"][:n_persons]
    assert np.array_equal(np.isnan(unit), np.isnan(r_unit))
    fin = ~np.isnan(r_unit)
    assert np.array_equal(unit[fin].view(np.int64), r_unit[fin].view(np.int64)), "unit lengths differ"
    present = got["present"][:n_persons]
    assert np.array_equal(present, r_present)
    for side in range(3):
        has = (present >> side & 1).astype(bool)
        assert np.array_equal(got["boxes"][:n_persons][has, side], r_boxes[has, side]), "side %d boxes differ" % side
    parts = got["parts"]
    assert [(int(p), int(sd)) for p, sd, _ in parts] == r_kept
    # the compacted tables: rows in order per kind, each the part's box, left hands mirrored
    rows = {0: 0, 1: 0}
    for person, side, row in parts:
        kind = 0 if side == 0 else 1
        assert row == rows[kind]
        rows[kind] += 1
        crop = (got["face"] if kind == 0 else got["hand"])[row]
        assert tuple(int(v) for v in (crop["left"], crop["top"], crop["right"], crop["bottom"])) == \
            tuple(int(v) for v in r_boxes[person, side])
        assert int(crop["flip"]) == int(side == 1)
    assert (rows[0], rows[1]) == (len(got["face"]), len(got["hand"]))
    return n_persons


def test_whole_body_boxes_batch_emulated(emu_lib, monkeypatch):
    native = pkg("_native")
    monkeypatch.setattr(native, "_lib", emu_lib)
    engine = native.Engine(0, pkg("pose_detector").make_opb_params())
    rs = np.random.RandomState(11)
    total = 0
    for s in (W.FRAME_SX, 1.0, 0.3):                       # 0.3: sub-pixel unit lengths, zero-width boxes
        frames = _batch(rs)
        got = _run(engine, frames, 320, s)
        assert len(got) == len(frames)
        total += sum(_check_frame(engine, g, fr, s) for g, fr in zip(got, frames))
    print("whole-body boxes, batch: %d persons checked" % total)
    assert total >= 3000


def test_whole_body_boxes_batch_range_error_is_per_frame(emu_lib, monkeypatch):
    """a box edge beyond int32 in one frame is that frame's status; the other frames are unaffected"""
    native = pkg("_native")
    monkeypatch.setattr(native, "_lib", emu_lib)
    engine = native.Engine(0, pkg("pose_detector").make_opb_params())
    rs = np.random.RandomState(5)
    far = W._records(1)
    W._put(far, 0, W.NOSE, 1 << 30, 5)
    W._put(far, 0, W.NECK, 0, 5)
    frames = [(1, 40, 0, W.random_persons(rs, 40)), (1, 1, 0, far), (1, 40, 0, W.random_persons(rs, 40))]
    got = _run(engine, frames, 64, 4.0)
    assert [g["status"] for g in got] == [0, native.ERR_UNSUPPORTED, 0]
    assert len(got[1]["parts"]) == 0
    _check_frame(engine, got[0], frames[0], 4.0)
    _check_frame(engine, got[2], frames[2], 4.0)
