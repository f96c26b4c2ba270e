"""Plain-Python harness shared by tests/test_gpu_conv_forms.py and tests/test_emu_conv_forms.py: runs single conv
launches of the pose, face and hand chains exactly as the chains build them (grouped problems, channel offsets,
concat-by-slice outputs, fp32 head maps, permuted Mconv1 weights, halved channel blocks) and checks every byte of the
output tensor they write.

Per launch (opb_test_chain_convs / opb_test_chain_conv_run):
  * inputs are drawn with a different scale per channel and encoded in the device layout of the precision (fast: fp16
    hi; parity: hi | lo fp16 planes; compensated: hi | per 64-channel chunk [e4m3(x_lo 2^11) x 64 | e4m3(x) x 64]);
    pad channels are zero, as in the chain;
  * the output tensor is prefilled with a sentinel byte whose fp16 and e4m3 readings are NaN; every byte the op does not
    own (channels outside [out_coff, out_coff + cout_valid) of each problem, and their lo / correction bytes) must still
    hold it afterwards;
  * every stored value is compared with a float64 conv2d of the decoded inputs with the layer's fp32 weights (reference
    channel order, independent of the library's permutation tables), + bias, ReLU, 2x2 max-pool, under a per-element
    bound a_p |ref| + b_p S + c_p, S = the element's own sum |x| (|w| + d_p) (see `bound_terms`);
  * where a problem also writes fp32 maps, the stored fp16 / lo / correction bytes must be exactly the encoding of the
    fp32 value (one epilogue produces both from the same float)."""
import collections

import numpy as np
import torch

from conftest import pkg

SENTINEL = 0x7F          # fp16 0x7F7F and e4m3 0x7F are both NaN
NETS = {"pose": ("models.CocoPoseNet", "CocoPoseNet"), "face": ("models.FaceNet", "FaceNet"),
        "hand": ("models.HandNet", "HandNet")}
PRECISIONS = ("fast", "parity", "comp")


def precision_id(native, prec):
    return {"fast": native.PRECISION_FAST, "parity": native.PRECISION_PARITY, "comp": native.PRECISION_COMP}[prec]


def make_engine(native, net, prec):
    """An Engine with the seeded He weights of `net` loaded in precision `prec`; returns (engine, {layer: (W, b)})."""
    modname, cls = NETS[net]
    nm = pkg(modname)
    syn = pkg("synthetic")
    wd = syn.he_weights(0) if net == "pose" else syn.he_weights(0, layers=nm.LAYERS)
    model = getattr(nm, cls)()
    model.load_npz(wd)
    eng = native.Engine(0, pkg("pose_detector").make_opb_params(), precision_id(native, prec))
    eng.load_model(model)
    weights = {k[:-2]: (wd[k].astype(np.float64), wd[k[:-2] + "/b"].astype(np.float64)) for k in wd if k.endswith("/W")}
    return eng, weights


# ---------------------------------------------------------------------------------------------------- launch forms
_PROB_FIELDS = ("in_h", "in_w", "in_c", "in_ctot", "in_coff", "out_h", "out_w", "out_c", "out_ctot", "out_coff",
                "cout_valid", "relu", "pool", "has_out32", "cin_pad", "cout_pad")


def signature(rec):
    """Every field of a launch record except the weights it multiplies (weight key, and with it the stage, and the
    weight-magnitude scale acc_scale): two launches with one signature run the same kernel variant, grid, channel
    offsets and store paths."""
    probs = tuple(tuple(int(rec["prob"][p][f]) for f in _PROB_FIELDS) for p in range(int(rec["n_problems"])))
    return (rec["tag"].decode(), int(rec["ks"]), int(rec["bn"]), int(rec["drain"]), int(rec["comp"]),
            int(rec["n_problems"]), int(rec["grid"]), int(rec["shared_in"])) + probs


def distinct_forms(recs):
    """signature -> index of its first launch, in launch order."""
    out = collections.OrderedDict()
    for i, r in enumerate(recs):
        out.setdefault(signature(r), i)
    return out


# ---------------------------------------------------------------------------------------------- reference layout
def _concat_map(dev_segments, ref_segments, width):
    """device channel -> reference channel of a concatenation, both given as ordered (name, channels) segments; -1 for
    the device's zero pad channels."""
    start, o = {}, 0
    for name, c in ref_segments:
        start[name] = (o, c)
        o += c
    m, o = np.full(width, -1, np.int64), 0
    for name, c in dev_segments:
        s, c2 = start[name]
        assert c2 == c
        m[o:o + c] = s + np.arange(c)
        o += c
    return m


def reference_of(net, wkey, weights, cin_pad):
    """(W [cout, cin_ref, k, k], b [cout], device input channel -> reference input channel [cin_pad]) of one packed
    weight key.  The stage-2..6 Mconv1 inputs are the concat tensor; the reference concatenates
    F.concat((h1, h2, feature_map)) (pose) / F.concat((h, feature_map)) (face, hand), the device stores
    [feature_map | PAF | heat | 0] / [feature_map | maps | 0] (DESIGN section 3)."""
    if wkey.endswith("_fused"):            # pose Mconv1: the L1 rows then the L2 rows, one N = 256 GEMM
        base = wkey[:-len("_fused")]
        (W1, b1), (W2, b2) = weights[base + "_L1"], weights[base + "_L2"]
        W, b = np.concatenate([W1, W2]), np.concatenate([b1, b2])
    else:
        W, b = weights[wkey]
    if wkey.startswith("Mconv1_"):
        if net == "pose":
            cmap = _concat_map([("feature", 128), ("paf", 38), ("heat", 19)], [("paf", 38), ("heat", 19), ("feature", 128)],
                               cin_pad)
        else:
            kc = W.shape[1] - 128
            cmap = _concat_map([("feature", 128), ("maps", kc)], [("maps", kc), ("feature", 128)], cin_pad)
    else:
        cmap = np.where(np.arange(cin_pad) < W.shape[1], np.arange(cin_pad), -1)
    assert sorted(cmap[cmap >= 0].tolist()) == list(range(W.shape[1]))
    return W, b, cmap


# ---------------------------------------------------------------------------------------------------- encodings
def e4m3_bytes(v):
    """e4m3 (fn) bytes of float32(v), round to nearest even, saturated to +-448 as __NV_SATFINITE does."""
    t = torch.from_numpy(np.clip(np.asarray(v, np.float32), -448.0, 448.0))
    return t.to(torch.float8_e4m3fn).view(torch.uint8).numpy()


def e4m3_values(b):
    return torch.from_numpy(np.ascontiguousarray(b, np.uint8)).view(torch.float8_e4m3fn).to(torch.float64).numpy()


def corr_byte_index(c):
    """byte of tensor channel c inside the correction plane of a pixel: [chunk c/64][x_lo 64 B | x 64 B]"""
    c = np.asarray(c)
    return (c // 64) * 128 + c % 64


def encode_input(x, prec):
    """x float64 [N, H, W, C] -> (raw uint8 [N, H, W, bytes per pixel], decoded float64 [N, H, W, C])."""
    x = np.clip(x, -448.0, 448.0)
    hi = x.astype(np.float16)
    hv = hi.astype(np.float64)
    if prec == "fast":
        return np.ascontiguousarray(hi).view(np.uint8), hv
    if prec == "parity":
        lo = (x - hv).astype(np.float16)
        return np.ascontiguousarray(np.concatenate([hi, lo], -1)).view(np.uint8), hv + lo.astype(np.float64)
    n, h, w, c = x.shape
    xl = e4m3_bytes((x - hv) * 2048.0)
    x8 = e4m3_bytes(x)
    corr = np.stack([xl.reshape(n, h, w, c // 64, 64), x8.reshape(n, h, w, c // 64, 64)], 4).reshape(n, h, w, 2 * c)
    raw = np.concatenate([np.ascontiguousarray(hi).view(np.uint8), corr], -1)
    return np.ascontiguousarray(raw), hv + e4m3_values(xl) / 2048.0


def draw_input(rs, n, h, w, c, zero_channels):
    """Per-channel scales 2^U(-2, 2) (a channel mix-up changes the result), magnitudes in [scale/2, 2 scale) with random
    signs: never tiny, so that the e4m3 copy of x has no subnormal floor (|x| >= 2^-3 > 2^-6)."""
    scale = 2.0 ** rs.uniform(-2, 2, c)
    mag = 2.0 ** rs.uniform(-1, 1, (n, h, w, c))
    x = np.where(rs.rand(n, h, w, c) < 0.5, -1.0, 1.0) * mag * scale
    x[..., zero_channels] = 0.0
    return x


# ---------------------------------------------------------------------------------------------------- error bounds
def n_pairs(rec, prec):
    chunks = int(rec["prob"][0]["cin_pad"]) // 64
    return chunks * {"fast": 1, "parity": 3, "comp": 2}[prec]


def bound_terms(rec, prec, p):
    """(a, b, c, d) of the per-element bound |stored - ref| <= a |ref| + b S + c, S = sum |x| (|w| + d) over the taps.

    Accumulation (all precisions): a wgmma k-step adds 16 products to the accumulator; aligned to the largest of the 17
    terms and truncated, each term loses less than one fp32 ulp (2^-23) of a partial sum, and every partial sum is at
    most S.  Two-level accumulation (parity, compensated) restarts the accumulator at every (chunk pair, filter column)
    step of ks taps x 4 k-steps and adds it to the running sum in round-to-nearest fp32, so a product passes through at
    most D = 17 * 4 ks + pairs * ks + 1 rounding events (the +1: the epilogue's fmaf with the bias); without it (fast)
    through D = 17 * 4 ks * ks * pairs + 1.  Accumulation error <= D 2^-23 S.
    fast       : operands are the fp16 values of the reference (products exact); output fp16 round to nearest:
                 a = 2^-11, c = 2^-25 (half the fp16 subnormal spacing).
    parity     : x = hi + lo exactly; W = Whi + Wlo up to Wlo's own fp16 rounding (2^-11 |W - Whi| <= 2^-22 |W|, or
                 2^-25 where Wlo is subnormal: d = 2^-25); the dropped lo * Wlo term <= 2^-11 2^-11 |x||W|.
                 Output hi + fp16(f - hi): a = 2^-22, c = 2^-25.
    compensated: x_hi * W_hi exact (fp16 products, exact power-of-two scaling 2^S); correction row x_lo e4m3(W 2^kW):
                 e4m3 rounds W by 2^-4, |x_lo| <= 2^-11 (1 + 2^-4) |x|  ->  2^-15 (1 + 2^-3) |x||W|;
                 e4m3(x) e4m3(W_lo 2^S): both rounded by 2^-4, |W_lo| <= 2^-11 |W|  ->  2^-11 (2^-3 + 2^-8) |x||W|;
                 the dropped x_lo W_lo <= 2^-22 (1 + 2^-3) |x||W|; the e4m3 subnormal floors (2^-10 in the scaled
                 units) give d = 2^-9 acc_scale.  Output hi + e4m3((f - hi) 2^11) / 2^11: a = 2^-4 2^-11 = 2^-15,
                 c = 2^-21 (the e4m3 subnormal floor 2^-10 / 2^11).
    a is applied to |ref| instead of |f|: |f| <= |ref| (1 + 2^-10) wherever the bound holds, covered by the factor 2."""
    ks = int(rec["ks"])
    pairs = n_pairs(rec, prec)
    if int(rec["drain"]):
        D = 17 * 4 * ks + pairs * ks + 1
    else:
        D = 17 * 4 * ks * ks * pairs + 1
    acc = D * 2.0 ** -23
    if prec == "fast":
        return 2 * 2.0 ** -11, acc, 2.0 ** -25, 0.0
    if prec == "parity":
        return 2 * 2.0 ** -22, acc + 2.0 ** -22 + 2.0 ** -22, 2.0 ** -25, 2.0 ** -25
    b = acc + 2.0 ** -15 * (1 + 2.0 ** -3) + 2.0 ** -11 * (2.0 ** -3 + 2.0 ** -8) + 2.0 ** -22 * (1 + 2.0 ** -3)
    return 2 * 2.0 ** -15, b, 2.0 ** -21, 2.0 ** -9 * float(rec["prob"][p]["acc_scale"])


# ------------------------------------------------------------------------------------------------------ reference
def reference(xdec, cmap, W, b, relu, pool, quantize, d, device):
    """float64 conv2d of the decoded input channels (device order -> reference order through cmap), + bias, ReLU,
    2x2 max-pool; and S = conv(|x|, |W| + d), max-pooled alike.  Returns NHWC arrays."""
    n, h, w, _ = xdec.shape
    X = torch.zeros((n, W.shape[1], h, w), dtype=torch.float64, device=device)
    dev = np.nonzero(cmap >= 0)[0]
    X[:, torch.from_numpy(cmap[dev])] = torch.from_numpy(np.ascontiguousarray(xdec[..., dev])).to(device).permute(0, 3, 1, 2)
    Wt = torch.from_numpy(W).to(device)
    if quantize:      # fast precision: the kernel multiplies the fp16 values of the operands (inputs already are)
        Wt = Wt.float().half().double()
    pad = (W.shape[2] - 1) // 2
    y = torch.nn.functional.conv2d(X, Wt, torch.from_numpy(b).to(device), padding=pad)
    S = torch.nn.functional.conv2d(X.abs(), Wt.abs() + d, None, padding=pad)
    if relu:
        y = torch.relu(y)
    if pool:
        assert relu
        y = torch.nn.functional.max_pool2d(y, 2, 2)
        S = torch.nn.functional.max_pool2d(S, 2, 2)
    return y.permute(0, 2, 3, 1).cpu().numpy(), S.permute(0, 2, 3, 1).cpu().numpy()


# ---------------------------------------------------------------------------------------------------------- a run
Result = collections.namedtuple("Result", "elements ratio")


def _written_mask(rec, prec, shape):
    """bytes of the output tensor the op owns"""
    q0 = rec["prob"][0]
    C = int(q0["out_c"])
    mask = np.zeros(shape[-1], bool)
    for p in range(int(rec["n_problems"])):
        q = rec["prob"][p]
        ch = int(q["out_coff"]) + np.arange(int(q["cout_valid"]))
        for plane in ([ch, C + ch] if prec == "parity" else [ch]):      # fp16 halves: hi (and lo)
            mask[2 * plane] = mask[2 * plane + 1] = True
        if prec == "comp":
            mask[2 * C + corr_byte_index(ch)] = True
            mask[2 * C + corr_byte_index(ch) + 64] = True
    return mask


def run_form(eng, net, prec, weights, n, h, w, index, rec, seed, device="cpu"):
    """Runs launch `index` of the (n, h, w) chain alone and checks it; returns Result(elements checked, largest
    err / bound)."""
    native = pkg("_native")
    rs = np.random.RandomState(seed)
    npb = int(rec["n_problems"])
    probs = [rec["prob"][p] for p in range(npb)]
    refs = [reference_of(net, rec["wkey"][p].decode(), weights, int(probs[p]["cin_pad"])) for p in range(npb)]
    # inputs: one tensor per distinct buffer; zero wherever a problem's reference has no channel (the chain's pad)
    n_in = 1 if (npb == 1 or int(rec["shared_in"])) else 2
    raws, decs = [], []
    for t in range(n_in):
        q = probs[t]
        C = int(q["in_c"])
        zero = np.zeros(C, bool)
        for p in range(npb):
            if n_in == 2 and p != t:
                continue
            c0, cmap = int(probs[p]["in_coff"]), refs[p][2]
            zero[c0 + np.nonzero(cmap < 0)[0]] = True
        x = draw_input(rs, n, int(q["in_h"]), int(q["in_w"]), C, zero)
        raw, dec = encode_input(x, prec)
        assert raw.shape[-1] == 2 * int(q["in_ctot"])
        raws.append(raw)
        decs.append(dec)
    q0 = probs[0]
    oh, ow, C, Ctot = (int(q0[f]) for f in ("out_h", "out_w", "out_c", "out_ctot"))
    out = np.full((n, oh, ow, 2 * Ctot), SENTINEL, np.uint8)
    out32 = [np.full((n, int(q["cout_valid"]), oh, ow), np.nan, np.float32) if int(q["has_out32"]) else None
             for q in probs] + [None] * (2 - npb)
    eng.test_chain_conv_run(n, h, w, index, raws[0], raws[1] if n_in == 2 else None, out, out32)

    # bytes the op does not own keep the sentinel
    mask = _written_mask(rec, prec, out.shape)
    stray = out[..., ~mask] != SENTINEL
    assert not stray.any(), "%s: %d bytes outside the written channels changed (first at byte %d of a pixel)" % (
        rec["tag"].decode(), int(stray.sum()), int(np.nonzero(~mask)[0][np.nonzero(stray.any((0, 1, 2)))[0][0]]))

    hi_all = out[..., :2 * C].view(np.float16)
    elements, worst = 0, 0.0
    for p in range(npb):
        q = probs[p]
        W, b, cmap = refs[p]
        cv, co, c0 = int(q["cout_valid"]), int(q["out_coff"]), int(q["in_coff"])
        xdec = decs[p if n_in == 2 else 0][..., c0:c0 + len(cmap)]
        a, bb, cc, d = bound_terms(rec, prec, p)
        ref, S = reference(xdec, cmap, W, b, int(q["relu"]), int(q["pool"]), prec == "fast", d, device)
        assert ref.shape == (n, oh, ow, cv)
        ch = co + np.arange(cv)
        hi = hi_all[..., ch]
        if prec == "fast":
            val = hi.astype(np.float64)
        elif prec == "parity":
            lo = out[..., 2 * C:4 * C].view(np.float16)[..., ch]
            val = hi.astype(np.float64) + lo.astype(np.float64)
        else:
            corr = out[..., 2 * C:]
            xl, x8 = corr[..., corr_byte_index(ch)], corr[..., corr_byte_index(ch) + 64]
            val = hi.astype(np.float64) + e4m3_values(xl) / 2048.0
            # the e4m3 copy of the value (the next layer's correction row): round to nearest of f, and f is within
            # 2^-15 |v| + 2^-21 of the decoded v
            vc = np.clip(val, -448.0, 448.0)
            ok8 = np.abs(e4m3_values(x8) - vc) <= (2.0 ** -4 + 2.0 ** -14) * np.abs(vc) + 2.0 ** -10
            assert ok8.all(), "%s problem %d: %d e4m3 value bytes off" % (rec["tag"].decode(), p, int((~ok8).sum()))
        bound = a * np.abs(ref) + bb * S + cc
        err = np.abs(val - ref)
        bad = ~(err <= bound)
        assert not bad.any(), "%s problem %d (%s): %d of %d values outside the bound; first at %s: %r vs ref %r (bound %r)" % (
            rec["tag"].decode(), p, prec, int(bad.sum()), bad.size, np.argwhere(bad)[0], val[bad][0], ref[bad][0], bound[bad][0])
        worst = max(worst, float((err / bound).max()))
        elements += err.size
        if out32[p] is not None:
            f = out32[p].transpose(0, 2, 3, 1)            # [N][cv][h][w] -> NHWC
            # fp32 maps: the same value before the output encoding (b S covers the accumulation and the fmaf)
            b32 = bb * S
            e32 = np.abs(f.astype(np.float64) - ref)
            assert (e32 <= b32).all(), "%s problem %d: fp32 maps outside the bound" % (rec["tag"].decode(), p)
            worst = max(worst, float((e32 / np.maximum(b32, 1e-300)).max()))
            elements += e32.size
            # exact encoding of the same fp32 value
            hi_f = f.astype(np.float16)
            assert np.array_equal(hi.view(np.uint16), hi_f.view(np.uint16)), "hi != fp16(out32)"
            rem = f - hi_f.astype(np.float32)                         # exact in fp32
            if prec == "parity":
                lo = out[..., 2 * C:4 * C].view(np.float16)[..., ch]
                assert np.array_equal(lo.view(np.uint16), rem.astype(np.float16).view(np.uint16)), "lo != fp16(f - hi)"
            elif prec == "comp":
                assert np.array_equal(xl, e4m3_bytes(rem * np.float32(2048.0))), "correction byte != e4m3((f - hi) 2^11)"
                assert np.array_equal(x8, e4m3_bytes(f)), "value byte != e4m3(f)"
    return Result(elements, worst)
