"""Write mc_parent_fingerprint.json: one deterministic training step of the sequence model (config A's shapes), the
token model (tiny), the masked-LM model (tiny, V = 1000) and the question-answering model (tiny), dropout on, under
torch.use_deterministic_algorithms -- the loss bits and a SHA-256 of the whole bf16 gradient space of each.  Run on
one H100 at the build before BertForMultipleChoice was added:

    python tests/golden/make_mc_parent_fingerprint.py tests/golden/mc_parent_fingerprint.json

tests/test_mc_regression.py recomputes the same fingerprints with `fingerprint` below and requires them bit for bit.
The sequence, token and masked-LM entries equal qa_parent_fingerprint.json's, which the script checks."""
import hashlib
import json
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

KINDS = ("sequence", "token", "mlm", "qa")


def fingerprint(kind):
    from parity import b2, tiny_config
    if kind == "sequence":
        cfg, cls = b2.chinese_bert_wwm_ext_config(num_labels=6), b2.BertForSequenceClassification
    elif kind == "token":
        cfg, cls = tiny_config(num_labels=9), b2.BertForTokenClassification
    elif kind == "mlm":
        cfg, cls = tiny_config(vocab_size=1000), b2.BertForMaskedLM
    else:
        cfg, cls = tiny_config(num_labels=2), b2.BertForQuestionAnswering
    torch.manual_seed(5)
    m = cls(cfg).cuda().train()
    m.set_dropout_rng_state(torch.tensor([11, 0]))
    if kind == "mlm":
        bt = b2.synthetic_mlm_batch(cfg, 8, 128, 3, padded=True)
    elif kind == "qa":
        bt = b2.synthetic_qa_batch(cfg, 8, 128, 3, padded=True)
    else:
        bt = b2.synthetic_batch(cfg, 8, 128, 3, padded=True)
    if kind == "token":
        lab = torch.randint(0, 9, (8, 128), generator=torch.Generator().manual_seed(4))
        lab[bt["attention_mask"] == 0] = -100
        bt["label"] = lab
    d = {k: v.cuda() for k, v in bt.items()}
    if kind == "qa":
        o = m(input_ids=d["input_ids"], token_type_ids=d["token_type_ids"], attention_mask=d["attention_mask"],
              start_positions=d["start_positions"], end_positions=d["end_positions"])
    else:
        o = m(input_ids=d["input_ids"], token_type_ids=d["token_type_ids"], attention_mask=d["attention_mask"],
              labels=d["label"])
    o.loss.backward()
    torch.cuda.synchronize()
    g = m._engine.grads.view(torch.int16).cpu().numpy().tobytes()
    return {"loss_bits": int(torch.tensor([float(o.loss.detach())]).view(torch.int32)),
            "grads_sha256": hashlib.sha256(g).hexdigest()}


def main(out):
    torch.use_deterministic_algorithms(True)
    try:
        got = {k: fingerprint(k) for k in KINDS}
    finally:
        torch.use_deterministic_algorithms(False)
    with open(os.path.join(HERE, "qa_parent_fingerprint.json")) as f:
        old = json.load(f)
    for k in ("sequence", "token", "mlm"):
        assert got[k] == old[k], (k, got[k], old[k])
    with open(out, "w") as f:
        json.dump(got, f)
    print(json.dumps(got))


if __name__ == "__main__":
    main(sys.argv[1])
