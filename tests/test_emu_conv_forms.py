"""CPU (`-m "not gpu"`): the conv launch forms that only the full chains build -- grouped two-problem launches with
per-problem input offsets, concat-by-slice outputs (PAF / heat / keypoint maps written into the concat tensor), fp32
head maps, the permuted Mconv1 weights and the halved channel block of small batches -- run one at a time on the
emulated library (tests/cuda_emu) and checked byte by byte by tests/conv_forms.py.  The dense single-problem forms of
the VGG front are what tests/test_emu_conv.py already runs; tests/test_gpu_conv_forms.py covers every form on the GPU.

176 x 64 is the smallest frame whose 1/8-resolution maps hold one 7x7 TMA box (22 x 8)."""
import ctypes as C
import os
import sys

import pytest

import conv_forms as F
from conftest import pkg

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "cuda_emu"))
import build_emu  # noqa: E402

SHAPE = (1, 176, 64)


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
def emu_native(emu_lib, monkeypatch):
    native = pkg("_native")
    monkeypatch.setattr(native, "_lib", emu_lib)
    # 3 "SMs": the persistent CTAs loop over many tiles, so every pipeline wraps
    monkeypatch.setenv("OPB_EMU_SMS", "3")
    return native


def _chain_only(rec):
    """a form opb_test_conv cannot build: two problems, a channel slice of a wider tensor, fp32 maps, or the concat
    (Mconv) layers"""
    q = rec["prob"][0]
    return (int(rec["n_problems"]) == 2 or int(q["out_c"]) != int(q["cout_valid"]) or int(q["has_out32"])
            or rec["tag"].decode().startswith("Mconv"))


def _run(native, net, prec, select):
    eng, weights = F.make_engine(native, net, prec)
    recs = eng.test_chain_convs(*SHAPE)
    ran = []
    for k, (sig, i) in enumerate(F.distinct_forms(recs).items()):
        if select(recs[i]):
            r = F.run_form(eng, net, prec, weights, *SHAPE, index=i, rec=recs[i], seed=k)
            assert r.ratio < 1.0
            ran.append(recs[i]["tag"].decode())
    return ran


@pytest.mark.parametrize("prec", ["parity", "comp"])
def test_pose_chain_forms(emu_native, prec):
    ran = _run(emu_native, "pose", prec, _chain_only)
    assert ran == ["conv4_4_CPM", "conv5_1", "conv5_2", "conv5_3", "conv5_4", "conv5_5", "Mconv1", "Mconv7x7", "Mconv6",
                   "Mconv7", "Mconv7"], ran      # Mconv7 twice: stages 2-5, and stage 6 with the fp32 maps


@pytest.mark.parametrize("prec", ["fast", "parity", "comp"])
@pytest.mark.parametrize("net", ["face", "hand"])
def test_keypoint_slice_and_head_forms(emu_native, net, prec):
    ran = _run(emu_native, net, prec, lambda r: int(r["prob"][0]["out_c"]) != int(r["prob"][0]["cout_valid"]))
    assert ran == ["conv5_3_CPM", "conv6_2_CPM", "Mconv7", "Mconv7"], ran


def test_pose_head_forms_fast(emu_native):
    """fast precision's own store paths (packed half2 pairs, scalar halves) on the PAF / heat slices of the concat"""
    ran = _run(emu_native, "pose", "fast", lambda r: r["tag"].decode() in ("conv5_5", "Mconv7"))
    assert ran == ["conv5_5", "Mconv7", "Mconv7"], ran


def test_small_batch_halved_forms(emu_native, monkeypatch):
    """With 132 SMs one frame fills less than a quarter wave and add_conv halves the channel block of the 7x7 launches
    (pose: the fused Mconv1 and the grouped Mconv2..5) to BN = 64; compensated precision runs the most epilogue planes."""
    monkeypatch.setenv("OPB_EMU_SMS", "132")
    ran = _run(emu_native, "pose", "comp", lambda r: int(r["bn"]) == 64 and int(r["ks"]) == 7)
    assert ran == ["Mconv1", "Mconv7x7"], ran
