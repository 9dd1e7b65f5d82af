"""The tensor-core decoder training kernel reproduces, bit for bit, the per-sample outputs recorded in
tests/golden/decoder_train_bits.npz (tests/golden/make_decoder_train_bits.py): sdf, d feats and the weight-gradient activation
buffer (dh1, the relu'(h2) words, d loss / d sdf), including that nothing is written past the sample count.  A change to how the
kernel schedules or stores its work must leave every one of these bits as they were."""
import sys

import numpy as np
import pytest

from util import G, golden

pytestmark = pytest.mark.gpu

sys.path.insert(0, G)
import make_decoder_train_bits as R  # noqa: E402


@pytest.fixture(scope="module")
def outputs():
    import torch
    import nerfloam_b200 as nl
    assert torch.cuda.is_available()
    return R.run_cases(nl)


def test_every_case_is_recorded(outputs):
    z = golden(R.NAME)
    want = {k[:-len("/sha256")] for k in z.files if k.endswith("/sha256")}
    got = {f"{case}/{name}" for case, arrays in outputs.items() for name in arrays}
    assert got == want


@pytest.mark.parametrize("case", ["ext_M300_wgrad1", "ext_M300_wgrad0", "ext_M16384_wgrad1", "ext_M16384_wgrad0", "ext_M16973_wgrad1",
                                  "ext_M16973_wgrad0", "loss_M16973_wgrad1", "loss_M16973_wgrad0", "count_M16973_n16800_wgrad1",
                                  "batch3_M16973"])
def test_outputs_equal_recorded_bits(outputs, case):
    z = golden(R.NAME)
    for name, t in outputs[case].items():
        key = f"{case}/{name}"
        if R.digest(t) == str(z[key + "/sha256"]):
            continue
        msg = f"{key}: digest differs"
        if key in z.files:      # the full recorded array: say where
            a, b = t.cpu().numpy().ravel(), z[key].ravel()
            diff = np.flatnonzero(a.view(np.uint32) != b.view(np.uint32))
            msg += f"; {diff.size} of {a.size} words differ, first at {diff[:8].tolist()}: got {a[diff[:4]]}, recorded {b[diff[:4]]}"
        pytest.fail(msg)
