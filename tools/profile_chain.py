"""Per-launch profile of one pose-network forward pass, set against what the hardware can do.

    python tools/profile_chain.py [--batch 32] [--height 368] [--width 656] [--precision comp]

Runs one batch of procedural frames through the pose pipeline to warm up, then once more with OPB_PROFILE=1 (a CUDA
event after every launch)
and prints, for each launch tag (grouped launches of one tag are summed):
  * the measured time;
  * the algorithmic FLOPs (2 x MACs of the reference layers, unpadded channel counts) and HBM bytes (each layer's
    input and output activations once in the precision's storage format, plus its weights), from the shapes;
  * the least time the hardware could take: the larger of FLOPs over the peak rate (fp32 CUDA cores for conv1_1,
    the dense fp16 tensor-core rate for every other conv) and bytes over the peak bandwidth, and which of the two
    bounds the launch;
  * the GPU name, power limit and SM clock, read in the same call.
Peaks come from MEASURED_PEAKS.json when it is present, else from NVIDIA's H100 SXM data sheet."""
import argparse
import json
import os
import re
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def peaks():
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.isfile(p):
        d = json.load(open(p))
        return dict(hbm_gbs=d["hbm_gbs"], fp16_tflops=d["bf16_tflops"], fp32_tflops=d.get("fp32_tflops", 67.0),
                    source="MEASURED_PEAKS.json" + ("" if "fp32_tflops" in d else " (fp32: data sheet)"))
    return dict(hbm_gbs=3350.0, fp16_tflops=989.0, fp32_tflops=67.0, source="H100 SXM data sheet (700 W)")


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=" + q, "--format=csv,noheader"],
                             stdout=subprocess.PIPE, text=True, timeout=10).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        out = "nvidia-smi unavailable: %s" % e
    return dict(zip(q.split(","), [s.strip() for s in out.split(",")])) if "," in out else {"error": out}


def layer_table(N, H, W, bpc):
    """tag -> list of (cin, cout, ks, h_in, w_in, h_out, w_out, in_bytes_per_px) of the pose chain (pool fused)."""
    h2, w2, h4, w4, h8, w8 = H // 2, W // 2, H // 4, W // 4, H // 8, W // 8
    t = {
        "conv1_1": [(3, 64, 3, H, W, H, W, 3)],                      # uint8 BGR frame in
        "conv1_2": [(64, 64, 3, H, W, h2, w2, None)],
        "conv2_1": [(64, 128, 3, h2, w2, h2, w2, None)],
        "conv2_2": [(128, 128, 3, h2, w2, h4, w4, None)],
        "conv3_1": [(128, 256, 3, h4, w4, h4, w4, None)],
        "conv3_2": [(256, 256, 3, h4, w4, h4, w4, None)],
        "conv3_3": [(256, 256, 3, h4, w4, h4, w4, None)],
        "conv3_4": [(256, 256, 3, h4, w4, h8, w8, None)],
        "conv4_1": [(256, 512, 3, h8, w8, h8, w8, None)],
        "conv4_2": [(512, 512, 3, h8, w8, h8, w8, None)],
        "conv4_3_CPM": [(512, 256, 3, h8, w8, h8, w8, None)],
        "conv4_4_CPM": [(256, 128, 3, h8, w8, h8, w8, None)],
        "conv5_1": [(128, 128, 3, h8, w8, h8, w8, None)] * 2,
        "conv5_2": [(128, 128, 3, h8, w8, h8, w8, None)] * 2,
        "conv5_3": [(128, 128, 3, h8, w8, h8, w8, None)] * 2,
        "conv5_4": [(128, 512, 1, h8, w8, h8, w8, None)] * 2,
        "conv5_5": [(512, 38, 1, h8, w8, h8, w8, None), (512, 19, 1, h8, w8, h8, w8, None)],
        "Mconv1": [(185, 128, 7, h8, w8, h8, w8, None)] * 2 * 5,
        "Mconv7x7": [(128, 128, 7, h8, w8, h8, w8, None)] * 2 * 4 * 5,
        "Mconv6": [(128, 128, 1, h8, w8, h8, w8, None)] * 2 * 5,
        "Mconv7": [(128, 38, 1, h8, w8, h8, w8, None), (128, 19, 1, h8, w8, h8, w8, None)] * 5,
    }
    out = {}
    for tag, layers in t.items():
        flops = byts = 0
        for cin, cout, ks, hi, wi, ho, wo, in_bpp in layers:
            flops += 2.0 * N * hi * wi * cin * cout * ks * ks
            byts += N * hi * wi * (in_bpp if in_bpp else cin * bpc) + N * ho * wo * cout * bpc
            byts += cout * cin * ks * ks * (4 if tag == "conv1_1" else bpc)
        out[tag] = (flops, byts)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--height", type=int, default=368)
    ap.add_argument("--width", type=int, default=656)
    ap.add_argument("--precision", default="comp", choices=["fast", "parity", "comp"])
    args = ap.parse_args()
    os.environ["OPB_PROFILE"] = "1"
    import __graft_entry__ as G
    pkg = G._pkg()
    native, syn = pkg._native, pkg.synthetic
    prec = {"fast": native.PRECISION_FAST, "parity": native.PRECISION_PARITY, "comp": native.PRECISION_COMP}[args.precision]
    model = G._pkg("models.CocoPoseNet").CocoPoseNet()
    model.load_npz(syn.he_weights(0))
    prm = G._pkg("pose_detector").make_opb_params(max_peaks=2048, max_candidates=8192, max_persons=64)
    eng = native.Engine(0, prm, precision=prec)
    eng.load_model(model)
    x = np.stack([syn.procedural_image(args.height, args.width, seed=i % 4) for i in range(args.batch)])
    run = lambda: eng.detect_batch(x, args.height, args.width)   # noqa: E731  (network-input-sized maps, as bench.py)

    def captured():   # the library reports the profile of each batch on stderr (fd 2)
        with tempfile.TemporaryFile(mode="w+") as tf:
            sys.stderr.flush()
            saved = os.dup(2)
            os.dup2(tf.fileno(), 2)
            try:
                run()
            finally:
                sys.stderr.flush()
                os.dup2(saved, 2)
                os.close(saved)
            tf.seek(0)
            return tf.read()

    captured()                                       # build the chain, load modules: this profile is discarded
    info = gpu_info()
    report = captured()
    info_after = gpu_info()
    rows = re.findall(r"\[opb profile\] (\S+)\s+n=\s*(\d+)\s+([\d.]+) ms", report)
    if not rows:
        sys.exit("no profile lines were reported:\n" + report)
    pk = peaks()
    bpc = 2 if args.precision == "fast" else 4
    table = layer_table(args.batch, args.height, args.width, bpc)
    print("GPU %s, power limit %s, SM clock %s before / %s after the pass (max %s); peaks: %s" % (
        info.get("name", "?"), info.get("power.limit", "?"), info.get("clocks.sm", "?"), info_after.get("clocks.sm", "?"),
        info.get("clocks.max.sm", "?"), pk["source"]))
    print("batch %d, %dx%d, %s precision" % (args.batch, args.height, args.width, args.precision))
    print("%-12s %4s %9s %9s %9s %9s %-7s %6s" % ("tag", "n", "ms", "GFLOP", "GB", "bound ms", "bound", "share"))
    total = 0.0
    res = []
    for tag, n, ms in rows:
        ms = float(ms)
        total += ms
        if tag not in table:
            print("%-12s %4s %9.3f %9s %9s %9s %-7s %6s" % (tag, n, ms, "-", "-", "-", "-", "-"))
            continue
        flops, byts = table[tag]
        rate = pk["fp32_tflops"] if tag == "conv1_1" else pk["fp16_tflops"]
        t_c, t_m = flops / (rate * 1e12) * 1e3, byts / (pk["hbm_gbs"] * 1e9) * 1e3
        bound = max(t_c, t_m)
        kind = ("fp32" if tag == "conv1_1" else "tensor") if t_c >= t_m else "HBM"
        print("%-12s %4s %9.3f %9.1f %9.3f %9.3f %-7s %5.1f%%" % (tag, n, ms, flops / 1e9, byts / 1e9, bound, kind,
                                                                   100.0 * bound / ms))
        res.append(dict(tag=tag, n=int(n), ms=ms, gflop=flops / 1e9, gb=byts / 1e9, bound_ms=bound, bound=kind))
    print("total %.3f ms" % total)
    print(json.dumps({"gpu": info, "gpu_after": info_after, "peaks": pk, "batch": args.batch, "height": args.height,
                      "width": args.width, "precision": args.precision, "total_ms": total, "launches": res}))


if __name__ == "__main__":
    main()
