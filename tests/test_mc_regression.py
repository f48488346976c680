"""GPU: adding the multiple-choice head changes nothing for the other models.  One training step of the sequence
model (config A's shapes), the token model (tiny), the masked-LM model (tiny) and the question-answering model (tiny),
dropout on, under torch.use_deterministic_algorithms: the loss bits and a SHA-256 of the whole bf16 gradient space must
equal what the build before BertForMultipleChoice produced (tests/golden/mc_parent_fingerprint.json, written on one
H100 by tests/golden/make_mc_parent_fingerprint.py, whose `fingerprint` this test runs)."""
import importlib.util
import json
import os

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "mc_parent_fingerprint.json")


def _maker():
    spec = importlib.util.spec_from_file_location("make_mc_parent_fingerprint",
                                                  os.path.join(HERE, "golden", "make_mc_parent_fingerprint.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["sequence", "token", "mlm", "qa"])
def test_one_step_matches_parent_bitwise(kind):
    with open(GOLDEN) as f:
        want = json.load(f)[kind]
    torch.use_deterministic_algorithms(True)
    try:
        got = _maker().fingerprint(kind)
    finally:
        torch.use_deterministic_algorithms(False)
    assert got == want
