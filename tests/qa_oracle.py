"""fp32 CPU restatement of HF ``BertForQuestionAnswering`` (eager attention) for the question-answering tests.

The encoder is oracle.bert_ref's (pinned against HF's BertForSequenceClassification by test_oracle.py); on top of the
last hidden state sits HF's qa_outputs, a Linear(H, 2) on every token with no dropout, split into start and end
logits, and HF's span loss: both positions clamped to [0, S], ``CrossEntropyLoss(ignore_index=S)`` over the sequence
axis for each, averaged.  `packed_span_loss` is the same loss with each sequence's softmax over its own tokens only
(HF's loss on every sequence run unpadded), which the packed path computes.  test_question_answering_cpu.py pins
this file against the installed transformers class.
"""
import torch
import torch.nn.functional as F

from parity import bert_ref


def hf_qa_model(cfg, seed=123):
    """HF BertForQuestionAnswering (eager attention, fp32, HF init under manual_seed(seed))"""
    from oracle import cpu_step
    from transformers import BertForQuestionAnswering
    torch.manual_seed(seed)
    return BertForQuestionAnswering(cpu_step.hf_config(cfg))


def qa_state_from_hf_init(cfg, seed=123):
    return {k: v.detach().clone() for k, v in hf_qa_model(cfg, seed).named_parameters()}


def span_loss(start_logits, end_logits, start_positions, end_positions):
    """HF BertForQuestionAnswering.forward's loss over [B, S] logits (transformers 5.5): squeeze [B, 1] positions,
    clamp both to [0, S], cross-entropy with ignore_index S for each, averaged"""
    if start_positions.dim() > 1:
        start_positions = start_positions.squeeze(-1)
    if end_positions.dim() > 1:
        end_positions = end_positions.squeeze(-1)
    ignored_index = start_logits.size(1)
    sp = start_positions.clamp(0, ignored_index)
    ep = end_positions.clamp(0, ignored_index)
    return (F.cross_entropy(start_logits, sp, ignore_index=ignored_index)
            + F.cross_entropy(end_logits, ep, ignore_index=ignored_index)) / 2


def packed_span_loss(start_logits, end_logits, attention_mask, start_positions, end_positions):
    """the packed path's loss restated on the padded [B, S] logits: each sequence's softmax over its valid tokens
    (padding logits -inf), HF's clamp and ignore rule with S the padded length"""
    pad = attention_mask == 0
    return span_loss(start_logits.masked_fill(pad, float("-inf")), end_logits.masked_fill(pad, float("-inf")),
                     start_positions, end_positions)


def forward(params, cfg, input_ids, token_type_ids=None, attention_mask=None, start_positions=None,
            end_positions=None, masks=None, packed=False):
    """(loss or None, start_logits [B, S], end_logits [B, S]).  masks: bert_ref's encoder keep masks (None: no
    dropout); the head has no dropout.  packed: the loss is packed_span_loss."""
    H = cfg.hidden_size
    P = dict(params)
    # bert_ref also runs the sequence head; a zero pooler and classifier feed it, and its logits are discarded
    P.setdefault("bert.pooler.dense.weight", torch.zeros(H, H))
    P.setdefault("bert.pooler.dense.bias", torch.zeros(H))
    P.setdefault("classifier.weight", torch.zeros(cfg.num_labels, H))
    P.setdefault("classifier.bias", torch.zeros(cfg.num_labels))
    _, _, x = bert_ref.forward(P, cfg, input_ids, token_type_ids, attention_mask, None, masks=masks,
                               return_hidden=True)
    logits = x @ P["qa_outputs.weight"].t() + P["qa_outputs.bias"]
    start, end = logits[..., 0], logits[..., 1]
    loss = None
    if start_positions is not None and end_positions is not None:
        if packed:
            loss = packed_span_loss(start, end, attention_mask, start_positions, end_positions)
        else:
            loss = span_loss(start, end, start_positions, end_positions)
    return loss, start, end


def loss_and_grads(params, cfg, batch, masks=None, packed=False):
    """one forward / backward of HF's span loss (or its packed restatement); grads keyed like `params`"""
    leaf = {k: v.detach().clone().requires_grad_(True) for k, v in params.items()}
    loss, start, end = forward(leaf, cfg, batch["input_ids"], batch.get("token_type_ids"),
                               batch.get("attention_mask"), batch["start_positions"], batch["end_positions"],
                               masks=masks, packed=packed)
    loss.backward()
    grads = {k: (v.grad if v.grad is not None else torch.zeros_like(v)) for k, v in leaf.items()}
    return loss.detach(), start.detach(), end.detach(), grads


def train(params, cfg, batches, lr=1e-3, weight_decay=0.01, packed=False):
    """HF AdamW over `batches` on one replica (dropout off); `params` are updated in place.  Returns the losses and
    the optimizer (its exp_avg moments)."""
    from oracle import adamw_ref
    opt = adamw_ref.HFAdamW(params, lr=lr, weight_decay=weight_decay)
    losses = []
    for b in batches:
        l, _s, _e, g = loss_and_grads(params, cfg, b, packed=packed)
        losses.append(l)
        opt.step(g)
    return torch.stack(losses), opt


def ddp_train(params, cfg, batches_per_step, lr=3e-5, weight_decay=0.01):
    """torch DDP over the QA model, restated: every rank's HF loss and gradients on its own batch, the gradients
    averaged over the ranks (the DDP all-reduce), one HF AdamW step.  Dropout off; `params` are updated in place.
    Returns per step dict(loss_mean) and, at the end, the optimizer."""
    from oracle import adamw_ref
    opt = adamw_ref.HFAdamW(params, lr=lr, weight_decay=weight_decay)
    history = []
    for rank_batches in batches_per_step:
        losses, grads = [], []
        for b in rank_batches:
            l, _s, _e, g = loss_and_grads(params, cfg, b)
            losses.append(l)
            grads.append(g)
        avg = {k: sum(g[k] for g in grads) / len(grads) for k in grads[0]}
        history.append({"loss_mean": torch.stack(losses).mean()})
        opt.step(avg)
    return history, opt
