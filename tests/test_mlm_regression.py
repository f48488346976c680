"""GPU: adding the masked-LM head changes nothing for the other models.  One training step of the sequence model
(config A's shapes) and of the token model (tiny), dropout on, under torch.use_deterministic_algorithms: the loss bits
and a SHA-256 of the whole bf16 gradient space must equal what the build before the masked-LM head produced
(tests/golden/mlm_parent_fingerprint.json)."""
import hashlib
import json
import os

import pytest
import torch

from parity import b2, tiny_config

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "mlm_parent_fingerprint.json")


def fingerprint(kind):
    cfg = tiny_config(num_labels=9) if kind == "token" else b2.chinese_bert_wwm_ext_config(num_labels=6)
    torch.manual_seed(5)
    cls = b2.BertForTokenClassification if kind == "token" else b2.BertForSequenceClassification
    m = cls(cfg).cuda().train()
    m.set_dropout_rng_state(torch.tensor([11, 0]))
    bt = b2.synthetic_batch(cfg, 8, 128, 3, padded=True)
    if kind == "token":
        lab = torch.randint(0, 9, (8, 128), generator=torch.Generator().manual_seed(4))
        lab[bt["attention_mask"] == 0] = -100
        bt["label"] = lab
    d = {k: v.cuda() for k, v in bt.items()}
    o = m(input_ids=d["input_ids"], token_type_ids=d["token_type_ids"], attention_mask=d["attention_mask"],
          labels=d["label"])
    o.loss.backward()
    torch.cuda.synchronize()
    g = m._engine.grads.view(torch.int16).cpu().numpy().tobytes()
    return {"loss_bits": int(torch.tensor([float(o.loss.detach())]).view(torch.int32)),
            "grads_sha256": hashlib.sha256(g).hexdigest()}


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["sequence", "token"])
def test_one_step_matches_parent_bitwise(kind):
    with open(GOLDEN) as f:
        want = json.load(f)[kind]
    torch.use_deterministic_algorithms(True)
    try:
        got = fingerprint(kind)
    finally:
        torch.use_deterministic_algorithms(False)
    assert got == want
