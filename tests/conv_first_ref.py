"""NumPy restatement of conv1_1 (preprocess + 3x3 conv 3 -> 64 + ReLU) down to the bytes of its output tensor.

Every output channel is `acc = bias; for r, s, c: acc = fmaf(x, w, acc)` in fp32.  One fmaf is restated exactly: the
float64 product of two floats is exact, TwoSum gives the float64 sum and its error, the sum is rounded to float32,
and when the float64 sum lies exactly halfway between two floats the sign of the error breaks the tie.  The output
encodings (fp16 hi, fp16 lo, 8-bit-float correction bytes) follow include/opb.h."""
import numpy as np

PIX_BYTES = {"fast": 128, "parity": 256, "comp": 256}


def fmaf(a, b, c):
    """Correctly rounded float32 a * b + c, elementwise (a, b, c float32 arrays that broadcast)."""
    p = a.astype(np.float64) * b.astype(np.float64)          # exact: 24 + 24 significant bits
    c64 = c.astype(np.float64)
    s = p + c64
    bb = s - p
    err = (p - (s - bb)) + (c64 - bb)                          # TwoSum: p + c == s + err exactly
    f = s.astype(np.float32)                                   # round half to even
    # s exactly halfway between two floats (25 significant bits: float64 mantissa bits 28..0 == 1 0...0; every value
    # here is far above float32's subnormal range): the exact sum lies on the side of err's sign
    mid = ((s.view(np.int64) & 0x1FFFFFFF) == 0x10000000) & (err != 0)
    if mid.any():
        idx = np.nonzero(mid)
        f[idx] = np.nextafter(s[idx], np.where(err[idx] > 0, np.inf, -np.inf)).astype(np.float32)
    return f


def preprocess_u8(x, denom):
    """uint8 [N,H,W,3] -> float32 [N,3,H,W]: float32(v) / denom - 0.5, both steps rounded in float32."""
    v = x.astype(np.float32) / np.float32(denom)
    return np.ascontiguousarray((v - np.float32(0.5)).astype(np.float32).transpose(0, 3, 1, 2))


def conv_first_acc(x_nchw, W, b, rows_per_chunk=64):
    """float32 [N,3,H,W] -> fp32 accumulators [N,H,W,64] before ReLU, in the kernel's exact fmaf order."""
    n, _, h, w = x_nchw.shape
    xp = np.zeros((n, 3, h + 2, w + 2), np.float32)
    xp[:, :, 1:-1, 1:-1] = x_nchw
    W = W.astype(np.float32)
    out = np.empty((n, h, w, 64), np.float32)
    for y0 in range(0, h, rows_per_chunk):
        y1 = min(h, y0 + rows_per_chunk)
        acc = np.broadcast_to(b.astype(np.float32), (n, y1 - y0, w, 64)).copy()
        for r in range(3):
            for s in range(3):
                for c in range(3):
                    xv = xp[:, c, y0 + r:y1 + r, s:s + w][..., None]
                    acc = fmaf(xv, W[:, c, r, s][None, None, None, :], acc)
        out[:, y0:y1] = acc
    return out


def e4m3(x):
    """float32 -> e4m3 bytes, round half to even, saturating at +-448 (NaN is not expected here)."""
    x = np.asarray(x, np.float32)
    a = np.abs(x).astype(np.float64)
    sign = np.where(np.signbit(x), 0x80, 0).astype(np.int64)
    q_sub = np.rint(a * 512.0).astype(np.int64)                # multiples of 2^-9 below 2^-6 (8 -> 2^-6 itself)
    m, e = np.frexp(np.where(a > 0, a, 1.0))
    E = e.astype(np.int64) - 1
    q = np.rint((2.0 * m - 1.0) * 8.0).astype(np.int64)
    E = np.where(q == 8, E + 1, E)
    q = np.where(q == 8, 0, q)
    norm = ((E + 7) << 3) | q
    norm = np.where((E + 7 > 15) | ((E + 7 == 15) & (q == 7)), 0x7E, norm)
    byte = np.where(a < 2.0 ** -6, q_sub, norm)
    return (byte | sign).astype(np.uint8)


def encode(acc, mode):
    """fp32 accumulators [N,H,W,64] -> raw output bytes [N,H,W,PIX_BYTES[mode]]."""
    v = np.maximum(acc, np.float32(0))
    hi = v.astype(np.float16)
    parts = [hi.view(np.uint8)]
    if mode != "fast":
        d = (v - hi.astype(np.float32)).astype(np.float32)    # exact
        if mode == "parity":
            parts.append(d.astype(np.float16).view(np.uint8))
        else:
            parts.append(e4m3(d * np.float32(2048.0)))
            parts.append(e4m3(v))
    return np.ascontiguousarray(np.concatenate(parts, axis=-1))


def make_weights(seed, scale=1.0):
    rs = np.random.RandomState(seed)
    W = (rs.standard_normal((64, 3, 3, 3)) * np.sqrt(2.0 / 27) * scale).astype(np.float32)
    b = (rs.standard_normal(64) * 0.1 * scale).astype(np.float32)
    b[b == 0] = np.float32(0.01)
    return W, b


def make_frame_u8(seed, n, h, w):
    """Random BGR frames with a saturated (255) band, a zero band and isolated 0 / 255 pixels."""
    rs = np.random.RandomState(seed)
    x = rs.randint(0, 256, (n, h, w, 3)).astype(np.uint8)
    x[:, : max(1, h // 6)] = 255
    x[:, h // 3: h // 3 + max(1, h // 6)] = 0
    x[:, :, : max(1, w // 8)] = 255
    x[:, :, -max(1, w // 9):] = 0
    m = rs.random_sample((n, h, w)) < 0.05
    x[m] = 255
    m = rs.random_sample((n, h, w)) < 0.05
    x[m] = 0
    return x


def make_frame_f32(seed, n, h, w):
    """Preprocessed float32 [N,3,H,W] in the preprocess range, with exact zeros and the extreme values."""
    rs = np.random.RandomState(seed)
    x = (rs.random_sample((n, 3, h, w)) - 0.5).astype(np.float32)
    x[:, :, : max(1, h // 5)] = np.float32(-0.5)
    x[:, :, h // 2: h // 2 + max(1, h // 7)] = np.float32(0)
    x[:, :, :, -max(1, w // 7):] = np.float32(255.0 / 255.0 - 0.5)
    return x
