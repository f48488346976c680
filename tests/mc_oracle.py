"""fp32 CPU restatement of HF ``BertForMultipleChoice`` (eager attention) for the multiple-choice tests.

HF's model flattens the [B, N, S] inputs to B·N sequences, runs BertModel with its pooler, dropout and a Linear(H, 1)
on each, and reads the [B·N, 1] logits as [B, N]; its loss is ``CrossEntropyLoss()`` over the N choices.  That is
oracle.bert_ref's sequence model (pinned against HF by test_oracle.py) with a one-row classifier on the flattened
rows, followed by the cross-entropy over the reshaped logits.  test_multiple_choice_cpu.py pins this file against the
installed transformers class.
"""
import torch
import torch.nn as nn

from parity import bert_ref


def hf_mc_model(cfg, seed=123):
    """HF BertForMultipleChoice (eager attention, fp32, HF init under manual_seed(seed))"""
    from oracle import cpu_step
    from transformers import BertForMultipleChoice
    torch.manual_seed(seed)
    return BertForMultipleChoice(cpu_step.hf_config(cfg))


def mc_state_from_hf_init(cfg, seed=123):
    return {k: v.detach().clone() for k, v in hf_mc_model(cfg, seed).named_parameters()}


def forward(params, cfg, input_ids, token_type_ids=None, attention_mask=None, labels=None, masks=None,
            criterion=None):
    """(loss or None, logits [B, N]).  masks: bert_ref's keep masks over the B·N flattened rows (None: no dropout).
    criterion: the loss over ([B, N] logits, [B] labels); None: HF's CrossEntropyLoss()."""
    B, N, S = input_ids.shape
    flat = lambda t: None if t is None else t.reshape(B * N, S)
    _, logits = bert_ref.forward(params, cfg, flat(input_ids), flat(token_type_ids), flat(attention_mask), None,
                                 masks=masks)
    logits = logits.view(B, N)
    loss = None
    if labels is not None:
        loss = (criterion or nn.CrossEntropyLoss())(logits, labels)
    return loss, logits


def loss_and_grads(params, cfg, batch, masks=None, criterion=None):
    """one forward / backward of the loss; grads keyed like `params`"""
    leaf = {k: v.detach().clone().requires_grad_(True) for k, v in params.items()}
    loss, logits = forward(leaf, cfg, batch["input_ids"], batch.get("token_type_ids"), batch.get("attention_mask"),
                           batch["label"], masks=masks, criterion=criterion)
    loss.backward()
    grads = {k: (v.grad if v.grad is not None else torch.zeros_like(v)) for k, v in leaf.items()}
    return loss.detach(), logits.detach(), grads


def train(params, cfg, batches, lr=1e-3, weight_decay=0.01):
    """HF AdamW over `batches` on one replica (dropout off); `params` are updated in place.  Returns the losses and
    the optimizer."""
    from oracle import adamw_ref
    opt = adamw_ref.HFAdamW(params, lr=lr, weight_decay=weight_decay)
    losses = []
    for b in batches:
        l, _logits, g = loss_and_grads(params, cfg, b)
        losses.append(l)
        opt.step(g)
    return torch.stack(losses), opt
