"""`-m gpu`: every distinct conv launch form of the CocoPoseNet, FaceNet and HandNet chains, run on its own on the
H100 and checked byte by byte (tests/conv_forms.py): per-element error bounds against a float64 reference, sentinel
bytes outside the written channels, exact hi / lo / correction encodings of the fp32 head maps.

Two (batch, frame) shapes per net: one image, where the grouped 7x7 launches (pose) or the 7x7 launches (face, hand)
fill less than a quarter wave and add_conv halves their channel block to BN = 64, and a batch where they keep
BN = 128.  176 x 128 is the smallest frame class whose 1/8-resolution maps hold one 7x7 TMA box (22 rows)."""
import numpy as np
import pytest
import torch

import conv_forms as F
from conftest import pkg

pytestmark = pytest.mark.gpu

SHAPES = {"pose": [(1, 176, 128), (5, 176, 128)], "face": [(1, 176, 128), (9, 176, 128)],
          "hand": [(1, 176, 128), (9, 176, 128)]}
# distinct launch forms of each chain at SHAPES on a 132-SM H100 (the same in all three precisions); a form added to
# the chain builders changes these counts, and the test then fails until the new form is checked here
EXPECTED_FORMS = {("pose", 1): 21, ("pose", 5): 21, ("face", 1): 24, ("face", 9): 24, ("hand", 1): 24, ("hand", 9): 24}


@pytest.mark.parametrize("prec", F.PRECISIONS)
@pytest.mark.parametrize("net", sorted(SHAPES))
def test_every_launch_form(net, prec):
    native = pkg("_native")
    eng, weights = F.make_engine(native, net, prec)
    device = "cuda" if torch.cuda.is_available() else "cpu"
    bns = set()
    elements, worst, n_forms = 0, 0.0, []
    for n, h, w in SHAPES[net]:
        recs = eng.test_chain_convs(n, h, w)
        forms = F.distinct_forms(recs)
        n_forms.append(len(forms))
        assert len(forms) == EXPECTED_FORMS[(net, n)], "%s at %s: %d launch forms" % (net, (n, h, w), len(forms))
        for k, (sig, i) in enumerate(forms.items()):
            r = F.run_form(eng, net, prec, weights, n, h, w, i, recs[i], seed=1000 * n + k, device=device)
            elements += r.elements
            worst = max(worst, r.ratio)
            if int(recs[i]["ks"]) == 7:
                bns.add(int(recs[i]["bn"]))
    # the two shapes reach both channel blocks of the 7x7 launches
    assert bns == {64, 128}, bns
    print("\n[conv forms] %s %s: forms %s, %d elements, max err/bound %.3g" % (net, prec, n_forms, elements, worst))
    assert worst < 1.0
