"""fp32 CPU restatement of HF ``BertForTokenClassification`` (eager attention) for the token-head tests.

The encoder is oracle.bert_ref's (pinned against HF's BertForSequenceClassification by test_oracle.py); on top of the
last hidden state sits the token head HF puts there: dropout (config.classifier_dropout, else hidden_dropout_prob)
and a linear classifier on every token, and ``CrossEntropyLoss(ignore_index)`` over ``logits.view(-1, C)``.
test_token_classification_cpu.py pins this file against the installed transformers class.
"""
import numpy as np
import torch
import torch.nn.functional as F

from parity import bert_ref, philox_keep_mask


def hf_token_model(cfg, seed=123):
    """HF BertForTokenClassification (eager attention, fp32, HF init under manual_seed(seed))"""
    from oracle import cpu_step
    from transformers import BertForTokenClassification
    torch.manual_seed(seed)
    return BertForTokenClassification(cpu_step.hf_config(cfg))


def token_state_from_hf_init(cfg, seed=123):
    return {k: v.detach().clone() for k, v in hf_token_model(cfg, seed).named_parameters()}


def classifier_p(cfg):
    p = getattr(cfg, "classifier_dropout", None)
    return float(p if p is not None else cfg.hidden_dropout_prob)


def token_head_mask(cfg, B, S, seed, step):
    """[B, S, H] keep mask of the token head's dropout: site 1 + 3 L, element (b S + s) H + h (b2_token_head_fwd)"""
    H, L = cfg.hidden_size, cfg.num_hidden_layers
    keep = philox_keep_mask(B * S * H, seed, step, 1 + 3 * L, classifier_p(cfg))
    return torch.from_numpy(np.ascontiguousarray(keep.reshape(B, S, H)))


def forward(params, cfg, input_ids, token_type_ids=None, attention_mask=None, labels=None, masks=None,
            head_mask=None, ignore_index=-100):
    """(loss or None, logits [B, S, C]).  masks: bert_ref's encoder keep masks (None: no dropout); head_mask: the
    [B, S, H] keep mask of the classifier dropout (None: none)."""
    H = cfg.hidden_size
    P = dict(params)
    # bert_ref also runs the sequence head; a zero pooler feeds it, and its logits are discarded
    P.setdefault("bert.pooler.dense.weight", torch.zeros(H, H))
    P.setdefault("bert.pooler.dense.bias", torch.zeros(H))
    seq_P = dict(P, **{"classifier.weight": P["classifier.weight"].detach(),
                       "classifier.bias": P["classifier.bias"].detach()})
    _, _, x = bert_ref.forward(seq_P, cfg, input_ids, token_type_ids, attention_mask, None, masks=masks,
                               return_hidden=True)
    p_c = classifier_p(cfg)
    if head_mask is not None and p_c > 0:
        x = x * head_mask.to(x.dtype) / (1.0 - p_c)
    logits = x @ P["classifier.weight"].t() + P["classifier.bias"]
    loss = None
    if labels is not None:
        loss = F.cross_entropy(logits.reshape(-1, cfg.num_labels), labels.reshape(-1), ignore_index=ignore_index)
    return loss, logits


def loss_and_grads(params, cfg, batch, masks=None, head_mask=None):
    """one forward / backward of HF's token loss; grads keyed like `params`"""
    leaf = {k: v.detach().clone().requires_grad_(True) for k, v in params.items()}
    loss, logits = forward(leaf, cfg, batch["input_ids"], batch.get("token_type_ids"), batch.get("attention_mask"),
                           batch["label"], masks=masks, head_mask=head_mask)
    loss.backward()
    grads = {k: (v.grad if v.grad is not None else torch.zeros_like(v)) for k, v in leaf.items()}
    return loss.detach(), logits.detach(), grads


def token_batch(cfg, batch, seq, seed, ignore_frac=0.15, min_len=8):
    """a right-padded tagging batch: ids ~ U{1..vocab-1} with [CLS] first, per-row lengths ~ U{min_len..seq}, labels
    ~ U{0..C-1} with -100 on padding, on [CLS] and on a random `ignore_frac` of the interior tokens (as a word-piece
    tagging collator leaves them)"""
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(1, cfg.vocab_size, (batch, seq), generator=g, dtype=torch.int64)
    ids[:, 0] = min(101, cfg.vocab_size - 1)
    lens = torch.randint(min_len, seq + 1, (batch,), generator=g)
    mask = (torch.arange(seq)[None] < lens[:, None]).to(torch.int64)
    ids = ids * mask
    lab = torch.randint(0, cfg.num_labels, (batch, seq), generator=g, dtype=torch.int64)
    drop = torch.rand(batch, seq, generator=g) < ignore_frac
    lab[drop | (mask == 0)] = -100
    lab[:, 0] = -100
    return {"input_ids": ids, "token_type_ids": torch.zeros_like(ids), "attention_mask": mask, "label": lab}


def ddp_train(params, cfg, batches_per_step, lr=3e-5, weight_decay=0.01):
    """torch DDP over the token model, restated: every rank's HF loss and gradients on its own batch, the gradients
    averaged over the ranks (the DDP all-reduce), one HF AdamW step.  Dropout off; `params` are updated in place.
    Returns per step dict(loss_mean) and, at the end, the optimizer (its exp_avg moments)."""
    from oracle import adamw_ref
    opt = adamw_ref.HFAdamW(params, lr=lr, weight_decay=weight_decay)
    history = []
    for rank_batches in batches_per_step:
        losses, grads = [], []
        for b in rank_batches:
            l, _z, g = loss_and_grads(params, cfg, b)
            losses.append(l)
            grads.append(g)
        avg = {k: sum(g[k] for g in grads) / len(grads) for k in grads[0]}
        history.append({"loss_mean": torch.stack(losses).mean()})
        opt.step(avg)
    return history, opt
