"""Reference side of the loss tests: the oracle's logits (oracle/bert_ref.forward) under HF's problem-type losses and
torch's criterion options, and labelled synthetic batches for each problem type."""
import torch
import torch.nn.functional as F

from parity import bert_ref


def hf_loss(logits, labels, problem_type, num_labels):
    """HF BertForSequenceClassification.forward's loss of a problem type (transformers 5.5)"""
    if problem_type == "regression":
        if num_labels == 1:
            return F.mse_loss(logits.squeeze(), labels.squeeze())
        return F.mse_loss(logits, labels)
    if problem_type == "single_label_classification":
        return F.cross_entropy(logits.view(-1, num_labels), labels.view(-1))
    return F.binary_cross_entropy_with_logits(logits, labels)


def criterion_loss(criterion, logits, labels):
    """a criterion applied as the package Trainer applies it: one label and float labels over the squeezed logits"""
    if logits.shape[-1] == 1 and labels.is_floating_point():
        return criterion(logits.reshape(-1), labels.reshape(-1))
    return criterion(logits, labels)


def loss_and_grads(params, cfg, batch, loss_fn):
    """oracle forward, loss_fn(logits, labels), backward: (loss, logits, grads by HF name)"""
    leaf = {k: v.detach().clone().requires_grad_(True) for k, v in params.items()}
    _, logits = bert_ref.forward(leaf, cfg, batch["input_ids"], batch.get("token_type_ids"),
                                 batch.get("attention_mask"), None)
    loss = loss_fn(logits, batch["label"])
    loss.backward()
    grads = {k: (v.grad if v.grad is not None else torch.zeros_like(v)) for k, v in leaf.items()}
    return loss.detach(), logits.detach(), grads


def labelled_batch(cfg, batch, seq, seed, kind, padded=True):
    """bert_ref.synthetic_batch with labels of `kind`: "single" int64 [batch], "regression" fp32 [batch] (one label) or
    [batch, C], "multi" {0, 1} fp32 [batch, C]"""
    b = bert_ref.synthetic_batch(cfg, batch, seq, seed, padded=padded)
    g = torch.Generator().manual_seed(seed + 77)
    C = cfg.num_labels
    if kind == "regression":
        b["label"] = torch.randn((batch,) if C == 1 else (batch, C), generator=g)
    elif kind == "multi":
        b["label"] = (torch.rand(batch, C, generator=g) < 0.4).to(torch.float32)
    return b
