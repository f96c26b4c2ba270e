"""`-m gpu`: conv1_1 (preprocess + 3x3 conv 3 -> 64 + ReLU) bit for bit against the NumPy restatement in
conv_first_ref.py, through opb_test_conv_first: all three precisions (fast, parity, compensated), uint8 frames
normalised by 255 (pose) and 256 (face / hand), preprocessed float32 input, sizes with partial tiles in both
directions, multi-image batches, and frames with saturated and zero pixels."""
import numpy as np
import pytest

import conv_first_ref as R
from conftest import pkg

pytestmark = pytest.mark.gpu

_PREC = {"fast": "PRECISION_FAST", "parity": "PRECISION_PARITY", "comp": "PRECISION_COMP"}

CASES = [
    # kind, denominator, n, h, w, weight scale
    ("u8", 255.0, 1, 37, 45, 1.0),
    ("u8", 255.0, 1, 368, 368, 1.0),
    ("u8", 255.0, 2, 368, 656, 1.0),
    ("u8", 256.0, 1, 37, 45, 1.0),
    ("u8", 256.0, 1, 368, 368, 1.0),
    ("f32", None, 1, 37, 45, 1.0),
    ("f32", None, 1, 368, 368, 1.0),
    ("u8", 255.0, 2, 9, 70, 300.0),     # activations past the largest e4m3 value (448): saturating correction bytes
    ("f32", None, 1, 1, 1, 1.0),        # a single pixel: every tap but the centre is padding
]

_cache = {}


def _case(case):
    if case not in _cache:
        kind, denom, n, h, w, scale = case
        seed = n * 100003 + h * 1009 + w + int(scale)
        W, b = R.make_weights(seed, scale)
        if kind == "u8":
            x = R.make_frame_u8(seed + 1, n, h, w)
            acc = R.conv_first_acc(R.preprocess_u8(x, denom), W, b)
        else:
            x = R.make_frame_f32(seed + 1, n, h, w)
            acc = R.conv_first_acc(x, W, b)
        _cache.clear()
        _cache[case] = (x, W, b, acc)
    return _cache[case]


@pytest.fixture(scope="module")
def native():
    return pkg("_native")


@pytest.fixture(scope="module")
def engine(native):
    return native.Engine(0, pkg("pose_detector").make_opb_params())


@pytest.mark.parametrize("mode", ["fast", "parity", "comp"])
@pytest.mark.parametrize("case", CASES, ids=lambda c: "%s%s_n%d_%dx%d_s%g" % (c[0], "" if c[1] is None else int(c[1]), *c[2:]))
def test_conv_first_bit_exact(engine, native, case, mode):
    x, W, b, acc = _case(case)
    denom = case[1] if case[1] is not None else 255.0
    got = engine.test_conv_first(x, W, b, getattr(native, _PREC[mode]), u8_denom=denom)
    ref = R.encode(acc, mode)
    assert got.shape == ref.shape
    bad = np.argwhere((got != ref).any(axis=-1))
    assert bad.size == 0, "%d of %d pixels differ, first at %s: got %s ref %s" % (
        len(bad), got.shape[0] * got.shape[1] * got.shape[2], bad[0].tolist(),
        got[tuple(bad[0])][:16].tolist(), ref[tuple(bad[0])][:16].tolist())


def test_conv_first_keeps_engine_weights(engine, native):
    """The hook runs with its own weights and leaves the context's conv1_1 and precision as they were."""
    img = pkg("synthetic").procedural_image(184, 184, seed=3)
    model = pkg("models.CocoPoseNet").CocoPoseNet()
    model.load_npz(pkg("synthetic").he_weights(0))
    det = pkg().PoseDetector(model=model, device=0, precision="parity")
    before = det.engine.forward(img[None])
    x, W, b, _ = _case(CASES[0])
    det.engine.test_conv_first(x, W, b, native.PRECISION_COMP)
    after = det.engine.forward(img[None])
    for p, q in zip(before, after):
        assert np.array_equal(p, q)
