"""HF's masked-language-model masking (``DataCollatorForLanguageModeling.torch_mask_tokens``, no whole-word masking)
for the inputs of ``BertForMaskedLM``: the same Bernoulli and ``randint`` draws, in the same order and on the same
shapes, so the same generator state gives the same masks bit for bit."""
import torch


def mask_tokens(input_ids, attention_mask=None, special_tokens_mask=None, *, mlm_probability=0.15,
                mask_replace_prob=0.8, random_replace_prob=0.1, mask_token_id=103, vocab_size, special_ids=(0, 101, 102),
                generator=None):
    """(inputs, labels) for masked-LM training, from int64 host ids [batch, seq].

    A position is chosen with probability `mlm_probability` unless it is special: its id is in `special_ids`
    ([PAD], [CLS], [SEP] of the BERT vocabularies), `attention_mask` is 0 there, or `special_tokens_mask` marks it.
    Labels are the original ids at chosen positions and -100 elsewhere.  Of the chosen positions, `mask_replace_prob`
    become `mask_token_id`, `random_replace_prob` a random id in [0, vocab_size), and the rest keep their id.
    `input_ids` is not modified; `generator` None draws from torch's default generator, as HF's does."""
    if not 0.0 <= mlm_probability <= 1.0:
        raise ValueError("mlm_probability=%r must be in [0, 1]" % (mlm_probability,))
    if mask_replace_prob < 0 or random_replace_prob < 0 or mask_replace_prob + random_replace_prob > 1:
        raise ValueError("mask_replace_prob=%r and random_replace_prob=%r must be non-negative and sum to at most 1"
                         % (mask_replace_prob, random_replace_prob))
    if input_ids.is_floating_point():
        raise TypeError("input_ids must be integer token ids, got %s" % input_ids.dtype)
    inputs = input_ids.clone()
    labels = input_ids.clone()
    special = torch.zeros(labels.shape, dtype=torch.bool)
    for sid in special_ids:
        special |= labels == int(sid)
    if attention_mask is not None:
        special |= attention_mask == 0
    if special_tokens_mask is not None:
        special |= special_tokens_mask.bool()
    probability_matrix = torch.full(labels.shape, mlm_probability)
    probability_matrix.masked_fill_(special, value=0.0)
    masked_indices = torch.bernoulli(probability_matrix, generator=generator).bool()
    labels[~masked_indices] = -100
    indices_replaced = torch.bernoulli(torch.full(labels.shape, mask_replace_prob), generator=generator).bool() \
        & masked_indices
    inputs[indices_replaced] = mask_token_id
    if mask_replace_prob == 1 or random_replace_prob == 0:
        return inputs, labels
    random_replace_prob_scaled = random_replace_prob / (1 - mask_replace_prob)
    indices_random = torch.bernoulli(torch.full(labels.shape, random_replace_prob_scaled), generator=generator).bool() \
        & masked_indices & ~indices_replaced
    random_words = torch.randint(vocab_size, labels.shape, dtype=torch.long, generator=generator)
    inputs[indices_random] = random_words[indices_random]
    return inputs, labels
