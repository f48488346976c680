"""fp32 CPU restatement of HF ``BertForMaskedLM`` (eager attention) for the masked-LM tests.

The encoder is oracle.bert_ref's (pinned against HF's BertForSequenceClassification by test_oracle.py); on top of the
last hidden state sits HF's cls.predictions: dense, erf GELU, LayerNorm, then the decoder tied to the word embeddings
plus cls.predictions.bias, and ``CrossEntropyLoss()`` over ``logits.view(-1, V)``.  test_masked_lm_cpu.py pins this
file against the installed transformers class.
"""
import torch
import torch.nn.functional as F

from parity import bert_ref


def hf_mlm_model(cfg, seed=123):
    """HF BertForMaskedLM (eager attention, fp32, HF init under manual_seed(seed))"""
    from oracle import cpu_step
    from transformers import BertForMaskedLM
    torch.manual_seed(seed)
    return BertForMaskedLM(cpu_step.hf_config(cfg))


def mlm_state_from_hf_init(cfg, seed=123):
    return {k: v.detach().clone() for k, v in hf_mlm_model(cfg, seed).named_parameters()}


def forward(params, cfg, input_ids, token_type_ids=None, attention_mask=None, labels=None, masks=None,
            ignore_index=-100):
    """(loss or None, logits [B, S, V]).  masks: bert_ref's encoder keep masks (None: no dropout); the head has no
    dropout."""
    H = cfg.hidden_size
    P = dict(params)
    # bert_ref also runs the sequence head; a zero pooler and classifier feed it, and its logits are discarded
    P.setdefault("bert.pooler.dense.weight", torch.zeros(H, H))
    P.setdefault("bert.pooler.dense.bias", torch.zeros(H))
    P.setdefault("classifier.weight", torch.zeros(cfg.num_labels, H))
    P.setdefault("classifier.bias", torch.zeros(cfg.num_labels))
    _, _, x = bert_ref.forward(P, cfg, input_ids, token_type_ids, attention_mask, None, masks=masks,
                               return_hidden=True)
    t = x @ P["cls.predictions.transform.dense.weight"].t() + P["cls.predictions.transform.dense.bias"]
    t = bert_ref.layer_norm(bert_ref.gelu_erf(t), P["cls.predictions.transform.LayerNorm.weight"],
                            P["cls.predictions.transform.LayerNorm.bias"], cfg.layer_norm_eps)
    logits = t @ P["bert.embeddings.word_embeddings.weight"].t() + P["cls.predictions.bias"]
    loss = None
    if labels is not None:
        loss = F.cross_entropy(logits.reshape(-1, cfg.vocab_size), labels.reshape(-1), ignore_index=ignore_index)
    return loss, logits


def loss_and_grads(params, cfg, batch, masks=None, dtype=torch.float32):
    """one forward / backward of HF's masked-LM loss; grads keyed like `params`"""
    leaf = {k: v.detach().to(dtype).clone().requires_grad_(True) for k, v in params.items()}
    loss, logits = forward(leaf, cfg, batch["input_ids"], batch.get("token_type_ids"), batch.get("attention_mask"),
                           batch["label"], masks=masks)
    loss.backward()
    grads = {k: (v.grad if v.grad is not None else torch.zeros_like(v)) for k, v in leaf.items()}
    return loss.detach(), logits.detach(), grads
