"""Decoder weight gradients at sample counts the gradient kernel's 64-sample chunking treats as edges, against fp64.

k_wgrad_tc splits the samples into 64-sample chunks dealt round-robin to nsplit CTAs per G tile (nsplit = SMs / 4, 33 on an
H100 SXM).  M = 77 leaves most CTAs without a chunk and ends in a partial chunk; M = 45 is less than one chunk.  The inputs,
the fp64 yardstick and the bar are those of test_gpu_decoder_wgrad.py."""
import pytest

from test_gpu_decoder_wgrad import BAR, fp64_grads, inputs, kernel_grads, rel_errors
from util import golden, load_decoder

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def setup():
    import torch
    import nerfloam_b200 as nl
    assert torch.cuda.is_available()
    return nl.engine, load_decoder(golden("render.npz"), "dec_")


@pytest.mark.parametrize("M", [77, 45])
def test_decoder_weight_gradients_at_chunking_edges_match_fp64(setup, M):
    E, dec = setup
    x, g = inputs(dec, M, seed=5)
    err = rel_errors(kernel_grads(E, dec, x, g, M), fp64_grads(dec, x, g))
    print(f"M={M} zeroed g: {int((g == 0).sum())}  errors vs fp64: " + " ".join(f"{n}={e:.2e}" for n, e in err.items()))
    assert all(e < BAR for e in err.values()), err
