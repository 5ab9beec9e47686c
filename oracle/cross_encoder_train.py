"""float64 CPU restatement of cross-encoder training: the grouped softmax cross-entropy of a one-label BERT or RoBERTa
sequence classifier, whose autograd gradient is the reference for the training tests.

  BERT     encode -> pooler dense -> tanh -> dropout -> classifier Linear          (BertForSequenceClassification)
  RoBERTa  encode -> dropout -> dense -> tanh -> dropout -> out_proj               (RobertaClassificationHead)
  loss     mean over groups of CrossEntropy(logits of the group's G pairs, label)

The body is oracle.encoder.encode.  Dropout is given as multipliers (keep / (1 - p), or 0): ``body`` as encode's
``dropout`` argument, ``head_in`` (RoBERTa's CLS rows before the dense layer) and ``head`` (after tanh) as [N, H]
tensors - the masks the CUDA path drew, replayed through dprb_dropout_mask (oracle/dropout.py restates them).
``head_ce`` is the part after the body, on given CLS rows.  ``sd`` holds CrossEncoder state_dict keys (oracle/cross_encoder.py).
"""
import torch
import torch.nn.functional as F

from .encoder import encode


def group_ce(sd, cfg, tokens, labels, G, body=None, head_in=None, head=None):
    """-> (loss float64 scalar, logits float64 [N])."""
    tokens = {k: torch.as_tensor(v) for k, v in tokens.items()}
    prefix = "transformer.roberta." if cfg.get("roberta", False) else "transformer.bert."
    cls = encode(sd, cfg, tokens, prefix=prefix, dropout=body)
    return head_ce(sd, cfg, cls, labels, G, head_in, head)


def head_ce(sd, cfg, cls, labels, G, head_in=None, head=None):
    """The classification head and the grouped cross-entropy on the body's CLS rows ``cls`` [N, H]
    -> (loss float64 scalar, logits float64 [N])."""
    if cfg.get("roberta", False):
        if head_in is not None:
            cls = cls * head_in
        dense, out = "transformer.classifier.dense.", "transformer.classifier.out_proj."
    else:
        dense, out = "transformer.bert.pooler.dense.", "transformer.classifier."
    t = torch.tanh(cls @ sd[dense + "weight"].T + sd[dense + "bias"])
    if head is not None:
        t = t * head
    logits = (t @ sd[out + "weight"].T + sd[out + "bias"]).reshape(-1)
    return F.cross_entropy(logits.view(-1, G), torch.as_tensor(labels, dtype=torch.int64)), logits
