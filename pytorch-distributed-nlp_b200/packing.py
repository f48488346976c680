"""Token packing for the reference's real input shape (§8 f3 of SURVEY.md).

The reference tokenises with ``padding="max_length", max_length=128`` (multi-gpu-distributed-cls.py:76) while the rows
of data/train.json average 18 characters: ~85 % of every [batch, 128] input is padding that the step still pays full
price for.  `pack_batch` re-arranges such a batch into fewer BINS of 128, 256, 384 or 512 tokens (`bin_length`: the
shortest that holds the batch's longest sequence): the valid prefixes of several sequences share one bin (first-fit,
longest first), every token keeps the position id it had in its own sequence, and every bin row carries the [lo, hi)
range of its own sequence inside the bin.  The attention kernels then mask with that range
(a block-diagonal mask per bin) instead of the key-padding mask, every other kernel is token-wise and simply sees
fewer rows, and the pooler reads each sequence's first token through `cls_index`.  Per sequence the arithmetic is
exactly that of the padded batch (a padded key contributes exp(-3.4e38 - m) = 0 to its softmax row, like a key of
another sequence here).  In bins longer than 128 tokens the attention kernels visit only the 128-token blocks a
sequence reaches, so a bin of short sequences costs little more than their tokens.
"""
import numpy as np
import torch

BIN = 128
MAX_BIN = 512      # the attention kernels' longest sequence


def bin_length(attention_mask, seq_len):
    """the bin length pack_batch should use for a [B, seq_len] (or multiple-choice [B, N, seq_len]) batch: the
    smallest multiple of BIN that holds its longest valid sequence (attention_mask None: every token is valid)"""
    longest = int(attention_mask.ne(0).sum(-1).max()) if attention_mask is not None else seq_len
    return BIN * max(1, -(-longest // BIN))


def pack_batch(input_ids, token_type_ids, attention_mask, bin_len=BIN, labels=None, ignore_index=-100,
               start_positions=None, end_positions=None):
    """input_ids / token_type_ids / attention_mask: int64 [B, S] host tensors as the reference's Collate yields them
    (valid tokens first: the tokenizer pads on the right).  Returns a dict of host tensors:
      input_ids, token_type_ids, position_ids   int64 [NB, bin_len]   (unused bin rows: pad id 0, position 0)
      segments                                   int32 [NB, bin_len]   lo | hi << 16: the row's own sequence is
                                                                       rows [lo, hi) of its bin (an unused row: itself)
      cls_index                                  int64 [B]             flat row (bin * bin_len + lo) of sequence b's
                                                                       first token, in the ORIGINAL batch order
      lengths                                    int64 [B]
      labels (when `labels`, int64 [B, S] token labels are given)
                                                 int64 [NB, bin_len]   unused bin rows: ignore_index
      start_positions, end_positions, seq_len    (when question-answering positions, int64 [B] or [B, 1], are
                                                 given) the positions as given, int64 [B] -- they count from each
                                                 sequence's first token, which packing keeps -- and S, HF's ignored
                                                 index.  A position in [length, S) targets a padding token, which
                                                 packing drops: ValueError.  Negative positions and positions >= S
                                                 pass through (the span loss clamps them as HF does).
    NB <= B; a sequence longer than bin_len is not supported (the reference truncates to max_seq_len = 128).
    A multiple-choice batch, int64 [B, N, S] tensors with `labels` int64 [B] (one choice index per example): the B·N
    choice sequences are packed as above, example-major; cls_index and lengths come back as [B, N] and the labels
    pass through as "labels"."""
    if input_ids.dim() == 3:
        return _pack_choices(input_ids, token_type_ids, attention_mask, bin_len, labels)
    if input_ids.dim() != 2:
        raise ValueError("input_ids must be [batch, seq] (or [batch, num_choices, seq])")
    B, S = input_ids.shape
    ids_np = input_ids.numpy()
    mask_np = (attention_mask.numpy() != 0) if attention_mask is not None else np.ones((B, S), dtype=bool)
    lens = mask_np.sum(1).astype(np.int64)
    # valid tokens must form a prefix (right padding): row i is exactly `lens[i]` ones followed by zeros
    if not np.array_equal(mask_np, np.arange(S)[None, :] < lens[:, None]):
        raise ValueError("pack_batch: attention_mask is not a right-padded prefix mask")
    if int(lens.min()) < 1:
        raise ValueError("pack_batch: empty sequence (no valid token)")
    if labels is not None:
        if labels.is_floating_point() or tuple(labels.shape) != (B, S):
            raise ValueError("pack_batch: labels must be int64 [%d, %d] token labels" % (B, S))
        lab_np = labels.numpy()
        # packing drops masked positions: a label there would vanish, where HF's loss would count it
        if bool((lab_np[~mask_np] != ignore_index).any()):
            raise ValueError("pack_batch: a masked position carries a label other than ignore_index=%d; packing drops "
                             "masked positions, so their labels must be ignored" % ignore_index)
    if (start_positions is None) != (end_positions is None):
        raise ValueError("pack_batch: start_positions and end_positions go together")
    qa = None
    if start_positions is not None:
        qa = []
        for t, nm in ((start_positions, "start_positions"), (end_positions, "end_positions")):
            if t.is_floating_point() or tuple(t.shape) not in ((B,), (B, 1)):
                raise ValueError("pack_batch: %s must be int64 [%d] or [%d, 1], got %s %s"
                                 % (nm, B, B, t.dtype, list(t.shape)))
            p = t.reshape(B).to(torch.int64)
            bad = (p >= torch.from_numpy(lens)) & (p < S)
            if bool(bad.any()):
                i = int(bad.nonzero()[0, 0])
                raise ValueError("pack_batch: %s[%d] = %d targets a padding token (the sequence has %d tokens, the batch "
                                 "%d): packing drops padding, so the target would vanish" % (nm, i, int(p[i]),
                                                                                             int(lens[i]), S))
            qa.append(p.clone())
    if int(lens.max()) > bin_len:
        raise ValueError("pack_batch: a sequence has %d valid tokens, more than the %d-token bin"
                         % (int(lens.max()), bin_len))
    # first-fit, longest first (ties in batch order): a few dozen integers -- plain Python
    ll = lens.tolist()
    order = sorted(range(B), key=lambda i: (-ll[i], i))
    free, bin_of, lo_of = [], [0] * B, [0] * B
    for i in order:
        n = ll[i]
        for k in range(len(free)):
            if free[k] >= n:
                bin_of[i], lo_of[i] = k, bin_len - free[k]
                free[k] -= n
                break
        else:
            free.append(bin_len - n)
            bin_of[i], lo_of[i] = len(free) - 1, 0
    NB = len(free)
    # one vectorised gather / scatter for all tokens
    lo = np.asarray(lo_of, dtype=np.int64)
    first = np.asarray(bin_of, dtype=np.int64) * bin_len + lo          # flat destination row of every sequence's [CLS]
    total = int(lens.sum())
    seq_of_tok = np.repeat(np.arange(B, dtype=np.int64), lens)
    starts = np.cumsum(lens) - lens
    within = np.arange(total, dtype=np.int64) - np.repeat(starts, lens)
    src = seq_of_tok * S + within
    dst = first[seq_of_tok] + within
    ids = np.zeros(NB * bin_len, dtype=np.int64)
    tts = np.zeros(NB * bin_len, dtype=np.int64)
    pos = np.zeros(NB * bin_len, dtype=np.int64)
    ar = np.arange(bin_len, dtype=np.int32)
    seg = np.tile(ar | ((ar + 1) << 16), NB)                             # unused rows: a segment of their own
    ids[dst] = ids_np.reshape(-1)[src]
    if token_type_ids is not None:
        tts[dst] = token_type_ids.numpy().reshape(-1)[src]
    pos[dst] = within
    seg[dst] = (lo[seq_of_tok] | ((lo[seq_of_tok] + lens[seq_of_tok]) << 16)).astype(np.int32)
    t = torch.from_numpy
    out = {"input_ids": t(ids).view(NB, bin_len), "token_type_ids": t(tts).view(NB, bin_len),
           "position_ids": t(pos).view(NB, bin_len), "segments": t(seg).view(NB, bin_len), "cls_index": t(first),
           "lengths": t(lens), "bins": NB}
    if labels is not None:
        lab = np.full(NB * bin_len, ignore_index, dtype=np.int64)
        lab[dst] = lab_np.reshape(-1)[src]
        out["labels"] = t(lab).view(NB, bin_len)
    if qa is not None:
        out["start_positions"], out["end_positions"], out["seq_len"] = qa[0], qa[1], S
    return out


def _pack_choices(input_ids, token_type_ids, attention_mask, bin_len, labels):
    """pack_batch of a [B, N, S] multiple-choice batch"""
    B, N, S = input_ids.shape
    for t, nm in ((token_type_ids, "token_type_ids"), (attention_mask, "attention_mask")):
        if t is not None and tuple(t.shape) != (B, N, S):
            raise ValueError("pack_batch: %s must have input_ids' shape %s, got %s" % (nm, [B, N, S], list(t.shape)))
    if labels is not None and (labels.is_floating_point() or tuple(labels.shape) != (B,)):
        raise ValueError("pack_batch: multiple-choice labels must be int64 [%d] (one choice index per example), got "
                         "%s %s" % (B, labels.dtype, list(labels.shape)))
    flat = lambda t: None if t is None else t.reshape(B * N, S)
    out = pack_batch(flat(input_ids), flat(token_type_ids), flat(attention_mask), bin_len)
    out["cls_index"] = out["cls_index"].view(B, N)
    out["lengths"] = out["lengths"].view(B, N)
    if labels is not None:
        out["labels"] = labels
    return out
