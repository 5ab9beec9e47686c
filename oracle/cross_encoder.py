"""float64 CPU restatement of the reference's CrossEncoder (dpr_scale/models/citadel_models/cross_encoder.py:21-26:
``AutoModelForSequenceClassification(**tokens).logits`` in eval mode).

  BERT     BertModel -> BertPooler (dense + tanh on token 0) -> dropout (identity) -> classifier Linear
           (site-packages/transformers/models/bert/modeling_bert.py: BertPooler, BertForSequenceClassification)
  RoBERTa  RobertaModel without pooler -> RobertaClassificationHead: token 0 -> dense -> tanh -> out_proj
           (site-packages/transformers/models/roberta/modeling_roberta.py)
The encoder body is oracle.encoder.encode.  ``sd`` holds the reference CrossEncoder's state_dict keys
(``transformer.bert.*`` + ``transformer.classifier.*``, or ``transformer.roberta.*`` + ``transformer.classifier.{dense,
out_proj}.*``).
"""
import torch

from .encoder import encode


def logits(sd, cfg, tokens):
    """cfg: oracle.encoder cfg keys (layers, heads, ln_eps, pad_id, roberta) -> logits float64 [N, num_labels]."""
    sd = {k: torch.as_tensor(v).double() if torch.as_tensor(v).is_floating_point() else torch.as_tensor(v)
          for k, v in sd.items()}
    tokens = {k: torch.as_tensor(v) for k, v in tokens.items()}
    if cfg.get("roberta", False):
        cls = encode(sd, cfg, tokens, prefix="transformer.roberta.")
        dense, out = "transformer.classifier.dense.", "transformer.classifier.out_proj."
    else:
        cls = encode(sd, cfg, tokens, prefix="transformer.bert.")
        dense, out = "transformer.bert.pooler.dense.", "transformer.classifier."
    h = torch.tanh(cls @ sd[dense + "weight"].T + sd[dense + "bias"])
    return h @ sd[out + "weight"].T + sd[out + "bias"]
