"""H100-native DDP BERT fine-tuning step behind the surface of taishan1994/pytorch-distributed-NLP's
``multi-gpu-distributed-cls.py``: same ``BertForSequenceClassification`` / ``DistributedDataParallel`` /
``build_optimizer`` / ``Trainer`` names, hand-written sm_90a kernels underneath (libb2ddpbert.so, C ABI in
include/b2_ddp_bert.h).  Importing never touches the GPU; the library is loaded (and required) on first use."""
from . import _lib
from .modeling import (BertConfig, BertForMaskedLM, BertForMultipleChoice, BertForQuestionAnswering,
                       BertForSequenceClassification, BertForTokenClassification, MultipleChoiceModelOutput,
                       QuestionAnsweringModelOutput, SequenceClassifierOutput, bert_base_config, bert_large_config,
                       chinese_bert_wwm_ext_config)
from .optim import SGD, Adam, AdamW, TorchAdamW, build_optimizer, clip_grad_norm_
from .ddp import DistributedDataParallel
from .synthetic import REFERENCE_LENGTH_HISTOGRAM, reference_length_batch, synthetic_batch, synthetic_mc_batch, \
    synthetic_mlm_batch, synthetic_qa_batch
from .masking import mask_tokens
from .packing import pack_batch
from .schedules import get_scheduler
from .losses import PROBLEM_TYPES, Loss, infer_problem_type, loss_from_criterion
from .trainer import Args, FusedEvalStep, FusedTrainStep, PackedTrainStep, Trainer


def set_seed(seed=123):
    """The reference's set_seed (multi-gpu-distributed-cls.py:17-26)."""
    import random
    import numpy as np
    import torch
    random.seed(seed)
    torch.manual_seed(seed)
    np.random.seed(seed)
    if torch.cuda.is_available():
        torch.cuda.manual_seed_all(seed)


__all__ = ["BertConfig", "BertForMaskedLM", "BertForQuestionAnswering", "QuestionAnsweringModelOutput",
           "synthetic_qa_batch", "BertForMultipleChoice", "MultipleChoiceModelOutput", "synthetic_mc_batch", "BertForSequenceClassification", "BertForTokenClassification", "mask_tokens",
           "synthetic_mlm_batch", "SequenceClassifierOutput", "AdamW", "SGD", "Adam", "TorchAdamW", "build_optimizer", "clip_grad_norm_",
           "DistributedDataParallel", "Args", "Trainer", "FusedTrainStep", "FusedEvalStep", "PackedTrainStep", "pack_batch", "get_scheduler", "Loss", "PROBLEM_TYPES", "infer_problem_type", "loss_from_criterion", "synthetic_batch", "reference_length_batch", "REFERENCE_LENGTH_HISTOGRAM", "set_seed", "bert_base_config",
           "bert_large_config", "chinese_bert_wwm_ext_config"]
