"""Synthetic inputs of the benchmark (SURVEY.md §8d; BASELINE.json `north_star`: no dataset, no tokenizer).

Stands in for what the reference's ``Collate.collate_fn`` yields (multi-gpu-distributed-cls.py:88-97): a dict of int64
host tensors ``input_ids / token_type_ids / attention_mask [batch, seq]`` and ``label [batch]``.
"""
import torch


def synthetic_batch(cfg, batch, seq, seed, padded=False, device="cpu"):
    """ids ~ U{0..vocab-1} with [:,0] = 101 (CLS), token types 0, labels ~ U{0..C-1}, generator seed `seed`;
    `padded` draws per-row valid lengths ~ U{8..seq} and zeroes ids / mask beyond them (the padded parity variant)."""
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(0, cfg.vocab_size, (batch, seq), generator=g, dtype=torch.int64)
    ids[:, 0] = min(101, cfg.vocab_size - 1)
    lab = torch.randint(0, cfg.num_labels, (batch,), generator=g, dtype=torch.int64)
    mask = torch.ones(batch, seq, dtype=torch.int64)
    if padded:
        lens = torch.randint(8, seq + 1, (batch,), generator=g)
        ar = torch.arange(seq)[None]
        mask = (ar < lens[:, None]).to(torch.int64)
        ids = ids * mask
    tt = torch.zeros(batch, seq, dtype=torch.int64)
    return {"input_ids": ids.to(device), "token_type_ids": tt.to(device), "attention_mask": mask.to(device),
            "label": lab.to(device)}


def synthetic_mlm_batch(cfg, batch, seq, seed, padded=False, mlm_probability=0.15):
    """synthetic_batch's dict for BertForMaskedLM: ids with [SEP] (102) closing each row, masked by masking.mask_tokens
    (its generator seeded from `seed`), and `label` the int64 [batch, seq] masked-LM labels (-100: not predicted)"""
    from .masking import mask_tokens
    b = synthetic_batch(cfg, batch, seq, seed, padded=padded)
    ids, mask = b["input_ids"], b["attention_mask"]
    last = mask.sum(1) - 1
    ids[torch.arange(batch), last] = min(102, cfg.vocab_size - 1)
    g = torch.Generator().manual_seed(seed + 1)
    inputs, labels = mask_tokens(ids, mask, mlm_probability=mlm_probability, mask_token_id=min(103, cfg.vocab_size - 1),
                                 vocab_size=cfg.vocab_size, generator=g)
    return {"input_ids": inputs, "token_type_ids": b["token_type_ids"], "attention_mask": mask, "label": labels}


def synthetic_qa_batch(cfg, batch, seq, seed, padded=False, no_answer=0.2, ignored=0.1, min_len=16):
    """A SQuAD-shaped batch for BertForQuestionAnswering, from generator seed `seed`: each row is [CLS] (101), 2 to 8
    question tokens (token type 0), [SEP] (102), context tokens (token type 1), [SEP]; `padded` draws per-row valid
    lengths ~ U{min_len..seq} (min_len >= 16) and zeroes ids / mask / token types beyond them.  start_positions <= end_positions lie inside
    the context; a `no_answer` fraction of rows is (0, 0) ([CLS], SQuAD v2's no answer) and an `ignored` fraction has a
    position >= seq (HF's loss clamps it to seq and ignores it).  Returns input_ids, token_type_ids, attention_mask,
    start_positions and end_positions (int64; the positions [batch])."""
    if not 16 <= min_len <= seq:
        raise ValueError("synthetic_qa_batch: need 16 <= min_len=%d <= seq=%d" % (min_len, seq))
    g = torch.Generator().manual_seed(seed)
    V = cfg.vocab_size
    ids = torch.randint(0, V, (batch, seq), generator=g, dtype=torch.int64)
    lens = torch.randint(min_len, seq + 1, (batch,), generator=g) if padded else torch.full((batch,), seq)
    qlen = torch.randint(2, 9, (batch,), generator=g)
    kind = torch.rand(batch, generator=g)
    u = torch.rand(batch, 3, generator=g)
    tt = torch.zeros(batch, seq, dtype=torch.int64)
    mask = (torch.arange(seq)[None] < lens[:, None]).to(torch.int64)
    start = torch.zeros(batch, dtype=torch.int64)
    end = torch.zeros(batch, dtype=torch.int64)
    cls_id, sep_id = min(101, V - 1), min(102, V - 1)
    for b in range(batch):
        n, q = int(lens[b]), int(qlen[b])
        ids[b, 0], ids[b, 1 + q], ids[b, n - 1] = cls_id, sep_id, sep_id
        tt[b, 2 + q:n] = 1
        lo, hi = 2 + q, n - 2                      # the context tokens, inclusive
        s = lo + int(u[b, 0] * (hi - lo + 1))
        e = s + int(u[b, 1] * min(hi - s + 1, 16))
        if kind[b] < no_answer:
            s = e = 0
        elif kind[b] < no_answer + ignored:
            over = seq + int(u[b, 2] * 8)
            if u[b, 2] < 0.5:
                s = over
            else:
                e = over
        start[b], end[b] = s, e
    ids = ids * mask
    return {"input_ids": ids, "token_type_ids": tt * mask, "attention_mask": mask, "start_positions": start,
            "end_positions": end}


def synthetic_mc_batch(cfg, batch, choices, seq, seed, padded=False):
    """A SWAG-shaped batch for BertForMultipleChoice, from generator seed `seed`: each of the `choices` rows of an
    example is [CLS] (101), the example's context (token type 0), [SEP] (102), that choice's ending and [SEP] (token
    type 1).  Every choice of an example shares its context.  `padded` draws the context length ~ U{2..seq/2 - 2} per
    example and each ending's length ~ U{1..seq - context - 3} per choice, and zeroes ids / mask / token types beyond
    them; otherwise the endings fill every row.  Returns input_ids, token_type_ids, attention_mask (int64 [batch,
    choices, seq]) and label (int64 [batch], the right choice)."""
    if seq < 8:
        raise ValueError("synthetic_mc_batch: need seq >= 8, got %d" % seq)
    g = torch.Generator().manual_seed(seed)
    V = cfg.vocab_size
    ids = torch.randint(0, V, (batch, choices, seq), generator=g, dtype=torch.int64)
    ctx = torch.randint(2, seq // 2 - 1, (batch,), generator=g)
    ctx_rows = ids[:, 0, :].clone()                  # one context per example, copied into each of its choices
    u = torch.rand(batch, choices, generator=g)
    lab = torch.randint(0, choices, (batch,), generator=g, dtype=torch.int64)
    tt = torch.zeros(batch, choices, seq, dtype=torch.int64)
    lens = torch.zeros(batch, choices, dtype=torch.int64)
    cls_id, sep_id = min(101, V - 1), min(102, V - 1)
    for b in range(batch):
        c = int(ctx[b])
        for k in range(choices):
            room = seq - c - 3
            end = 1 + int(u[b, k] * room) if padded else room
            n = c + end + 3
            ids[b, k, 1:1 + c] = ctx_rows[b, 1:1 + c]
            ids[b, k, 0], ids[b, k, 1 + c], ids[b, k, n - 1] = cls_id, sep_id, sep_id
            tt[b, k, 2 + c:n] = 1
            lens[b, k] = n
    mask = (torch.arange(seq)[None, None] < lens[..., None]).to(torch.int64)
    return {"input_ids": ids * mask, "token_type_ids": tt * mask, "attention_mask": mask, "label": lab}


# Token-length histogram of the reference's own data (data/train.json, 40 133 rows): characters of the text without the
# segmentation blanks (BertTokenizer splits Chinese text into single characters) + [CLS] + [SEP], capped at
# max_seq_len = 128 (multi-gpu-distributed-cls.py:66-98).  (length, rows); mean 19.8 tokens -- the reference pads all of
# them to 128 (`padding="max_length"`, :76).
REFERENCE_LENGTH_HISTOGRAM = (
    (3, 7), (4, 122), (5, 324), (6, 583), (7, 1493), (8, 2600), (9, 2580), (10, 2416), (11, 2277), (12, 2160),
    (13, 1991), (14, 1920), (15, 1758), (16, 1529), (17, 1489), (18, 1381), (19, 1296), (20, 1148), (21, 1061),
    (22, 956), (23, 875), (24, 748), (25, 726), (26, 657), (27, 588), (28, 585), (29, 517), (30, 439), (31, 394),
    (32, 384), (33, 331), (34, 330), (35, 300), (36, 236), (37, 241), (38, 185), (39, 184), (40, 189), (41, 155),
    (42, 146), (43, 161), (44, 150), (45, 129), (46, 134), (47, 114), (48, 106), (49, 102), (50, 103), (51, 107),
    (52, 83), (53, 78), (54, 72), (55, 64), (56, 70), (57, 78), (58, 68), (59, 65), (60, 57), (61, 56), (62, 51),
    (63, 55), (64, 45), (65, 42), (66, 39), (67, 44), (68, 51), (69, 29), (70, 27), (71, 27), (72, 32), (73, 38),
    (74, 28), (75, 26), (76, 21), (77, 30), (78, 21), (79, 22), (80, 14), (81, 20), (82, 24), (83, 11), (84, 21),
    (85, 15), (86, 18), (87, 18), (88, 15), (89, 12), (90, 13), (91, 10), (92, 10), (93, 11), (94, 9), (95, 12),
    (96, 8), (97, 7), (98, 5), (99, 8), (100, 10), (101, 8), (102, 9), (103, 6), (104, 3), (105, 8), (106, 4),
    (107, 7), (108, 10), (109, 7), (110, 4), (111, 3), (112, 4), (113, 5), (114, 3), (115, 6), (116, 3), (117, 5),
    (118, 3), (119, 3), (120, 2), (121, 3), (122, 2), (123, 7), (124, 2), (126, 1), (127, 2), (128, 16))


def reference_length_batch(cfg, batch, seed, seq=128):
    """A batch shaped like the reference's real input: valid lengths drawn from REFERENCE_LENGTH_HISTOGRAM, ids random,
    right-padded to `seq` with id 0 / mask 0 exactly as the reference's tokenizer call pads (:76)."""
    g = torch.Generator().manual_seed(seed)
    lengths = torch.tensor([l for l, _ in REFERENCE_LENGTH_HISTOGRAM], dtype=torch.int64)
    weights = torch.tensor([float(c) for _, c in REFERENCE_LENGTH_HISTOGRAM])
    lens = lengths[torch.multinomial(weights, batch, replacement=True, generator=g)].clamp(max=seq)
    ids = torch.randint(1, cfg.vocab_size, (batch, seq), generator=g, dtype=torch.int64)
    ids[:, 0] = min(101, cfg.vocab_size - 1)
    mask = (torch.arange(seq)[None] < lens[:, None]).to(torch.int64)
    lab = torch.randint(0, cfg.num_labels, (batch,), generator=g, dtype=torch.int64)
    return {"input_ids": ids * mask, "token_type_ids": torch.zeros(batch, seq, dtype=torch.int64),
            "attention_mask": mask, "label": lab}
