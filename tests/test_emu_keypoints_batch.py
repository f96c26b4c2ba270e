"""CPU (`-m "not gpu"`): opb_keypoints_detect_crops -- every face / hand crop of a frame in one device pass -- run under
the CPU emulation of tests/cuda_emu (see tests/test_emu_conv.py), against the per-crop path on the same engine.

FaceNet in fast precision at a network size of 176 (the smallest the 7x7 TMA boxes admit; the emulated tensor core makes
every image of a forward cost about a minute and a half).  The default run checks one crop that is partly outside the
frame, mirrored and downscaled (two forwards); the four-crop chunk -- partly outside and mirrored, larger than the
network input, entirely outside, tiny -- with its four per-crop references is opt-in (OPB_TEST_SLOW=1, eight forwards).
Multi-chunk calls (more than 16 crops) and 40-crop bit identity are covered on the GPU (tests/test_gpu_keypoints_batch.py)."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

from conftest import pkg

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "cuda_emu"))
import build_emu  # noqa: E402

NET = 176
THRESH = 0.1


@pytest.fixture(scope="module")
def emu_lib():
    native = pkg("_native")
    try:
        lib = C.CDLL(build_emu.build(contract=False))
    except (RuntimeError, OSError) as e:     # no g++ / CUDA headers on this box: the harness, not the product, is missing
        pytest.skip("emulated build unavailable: %s" % str(e)[:200])
    for name, (res, args) in native._SIGNATURES.items():
        fn = getattr(lib, name)
        fn.restype = res
        fn.argtypes = args
    return lib


@pytest.fixture()
def face_det(emu_lib, monkeypatch):
    native, entity, syn = pkg("_native"), pkg("entity"), pkg("synthetic")
    monkeypatch.setattr(native, "_lib", emu_lib)
    monkeypatch.setitem(entity.params, "face_inference_img_size", NET)
    monkeypatch.setitem(entity.params, "face_heatmap_peak_thresh", THRESH)
    nm = pkg("models.FaceNet")
    net = nm.FaceNet()
    net.load_npz(syn.he_weights(0, layers=nm.LAYERS))
    return pkg("face_detector").FaceDetector(model=net, device=0, precision="fast")


def _same(a, b):
    """keypoint lists equal bit for bit: validity, x, y, float32 confidence and element types"""
    assert len(a) == len(b)
    for ka, kb in zip(a, b):
        assert (ka is None) == (kb is None), (ka, kb)
        if ka is not None:
            assert type(ka[0]) is int and type(ka[1]) is int and isinstance(ka[2], np.float32)
            assert (ka[0], ka[1]) == (kb[0], kb[1]) and np.float32(ka[2]).tobytes() == np.float32(kb[2]).tobytes(), (ka, kb)


CROP_SETS = {
    # one crop that is partly outside the frame (left edge), mirrored like a left hand and larger than the network input
    "one": [(-40, 30, 160, 230, 1)],
    "four": [(-30, 100, 50, 190, 1),     # partly outside the frame (left edge), mirrored like a left hand
             (60, 20, 270, 230, 0),      # 210 x 210: larger than the network input (downscale)
             (400, 300, 450, 340, 0),    # entirely outside: an all-zero canvas
             (10, 10, 17, 15, 0)],       # 5 x 7
}
_SLOW = pytest.mark.skipif(os.environ.get("OPB_TEST_SLOW", "0") != "1",
                           reason="eight emulated forwards, about 14 minutes: set OPB_TEST_SLOW=1")


@pytest.mark.parametrize("name", ["one", pytest.param("four", marks=_SLOW)])
def test_detect_crops_equals_per_crop_path(face_det, name):
    import cv2
    det, eng = face_det, face_det.engine
    crop_image = pkg("pose_detector").PoseDetector.crop_image
    frame = pkg("synthetic").procedural_image(240, 320, seed=31)
    crops = CROP_SETS[name]
    l0 = eng.launch_count()
    got = eng.keypoints_detect_crops(frame, crops, NET, THRESH)
    per_chunk = eng.launch_count() - l0
    assert len(got) == len(crops)
    per_crop = []
    for (l, t, r, b, flip), kps in zip(crops, got):
        canvas = crop_image(None, frame, (l, t, r, b))
        l0 = eng.launch_count()
        if flip:      # HandDetector.__call__(canvas, hand_type="left")
            ref = eng.keypoints_detect(cv2.flip(canvas, 1), NET, THRESH, mirror=True)
        else:
            ref = det(canvas)
        per_crop.append(eng.launch_count() - l0)
        assert len(kps) == 70 and sum(k is not None for k in ref) > 0
        _same(kps, ref)
    # the crops share one forward chunk: as many launches as ONE per-crop call that needs a resize (resize, chain,
    # upsample, two smoothing passes, arg-max), whatever the number of crops in the chunk
    assert per_chunk == per_crop[-1] and sum(per_crop) == len(crops) * per_chunk


def test_detect_crops_rejects_empty_crops_before_launching(face_det):
    det, eng = face_det, face_det.engine
    native = pkg("_native")
    frame = np.zeros((40, 60, 3), np.uint8)
    l0 = eng.launch_count()
    for bad in ([(5, 5, 5, 20)], [(0, 0, 10, 10), (3, 9, 20, 4)], [(0, 0, 10)], [(0.0, 0, 10, 10)]):
        with pytest.raises(ValueError):
            det.detect_crops(frame, bad)
    # the C entry point itself refuses the crop (OPB_ERR_ARG) without launching anything
    table = np.zeros(2, native.CROP_DTYPE)
    table[0] = (0, 0, 8, 8, 0, 0)
    table[1] = (4, 4, 12, 4, 0, 0)
    with pytest.raises(native.OpbError, match="-2"):
        eng.keypoints_detect_crops(frame, table, NET, THRESH)
    assert det.detect_crops(frame, []) == []
    assert eng.launch_count() == l0
