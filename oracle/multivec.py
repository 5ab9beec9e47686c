"""float64 CPU restatement of the reference's COIL and CITADEL reranking paths:

  coil         dpr_scale/models/citadel_models/coil_model.py:45-61: hidden_states[-1][:, 1:] -> project -> * mask; ids =
               input_ids[:, 1:], weights = attention_mask[:, 1:]; cls_repr = cls_project(hidden_states[-1][:, 0])
  citadel      dpr_scale/models/citadel_models/citadel_model.py:46-82: router logits = the masked-LM head on
               hidden_states[-1][:, 1:] (BERT: cls.predictions.transform = dense -> gelu -> LayerNorm, then the decoder
               tied to the word embeddings + cls.predictions.bias; RoBERTa / XLM-R: lm_head.{dense, layer_norm, decoder,
               bias}), full_router_repr = log(1 + relu(logits)) * mask, (weights, ids) = topk(full_router_repr, k),
               expert_repr = tok_project(hidden_states[-1][:, 1:]) * mask
  expert_score dpr_scale/task/citadel_eval_task.py:238-265 with expert ids (both branches), plus the CLS term of
               _eval_step (:282-283)
The encoder layers are oracle.encoder's (through oracle.colbert.hidden_states).  ``sd`` holds an encoder's state_dict
keys under ``prefix``.
"""
import torch

from .colbert import _double, hidden_states, project
from .encoder import gelu_erf, layer_norm


def _linear(sd, x, prefix):
    """A ``Sequential(Linear)`` projection (``prefix`` + ``0.weight``), or the identity without one."""
    return project(sd, x, prefix)


def coil(sd, cfg, tokens, add_cls=False, prefix=""):
    """COILEncoder.forward(tokens, add_cls) in float64."""
    h = hidden_states(sd, cfg, tokens, prefix + "transformer.")
    am = torch.as_tensor(tokens["attention_mask"])
    out = {"expert_repr": _linear(sd, h[:, 1:], prefix + "project.") * am[:, 1:].unsqueeze(-1).double(),
           "expert_ids": torch.as_tensor(tokens["input_ids"])[:, 1:].clone(),
           "expert_weights": am[:, 1:].clone(), "attention_mask": am[:, 1:].clone()}
    if add_cls:
        out["cls_repr"] = _linear(sd, h[:, 0], prefix + "cls_project.")
    return out


def head_kind(sd, prefix=""):
    """'bert' (transformer.bert.* + cls.predictions.*) or 'roberta' (transformer.roberta.* + lm_head.*)."""
    return "bert" if prefix + "transformer.cls.predictions.bias" in sd else "roberta"


def router_logits(sd, h, ln_eps, prefix=""):
    """The masked-LM head of a CITADEL encoder on hidden states h [..., H] -> float64 logits [..., V]."""
    sd = _double(sd)
    t = prefix + "transformer."
    if head_kind(sd, prefix) == "bert":
        p = t + "cls.predictions."
        x = gelu_erf(h @ sd[p + "transform.dense.weight"].T + sd[p + "transform.dense.bias"])
        x = layer_norm(x, sd[p + "transform.LayerNorm.weight"], sd[p + "transform.LayerNorm.bias"], ln_eps)
        word, bias = sd[t + "bert.embeddings.word_embeddings.weight"], sd[p + "bias"]
    else:
        p = t + "lm_head."
        x = gelu_erf(h @ sd[p + "dense.weight"].T + sd[p + "dense.bias"])
        x = layer_norm(x, sd[p + "layer_norm.weight"], sd[p + "layer_norm.bias"], ln_eps)
        word, bias = sd[t + "roberta.embeddings.word_embeddings.weight"], sd[p + "bias"]
    return x @ word.T + bias


def citadel(sd, cfg, tokens, topk=1, add_cls=False, prefix=""):
    """CITADELEncoder.forward(tokens, topk, add_cls) in float64, without the training statistics.  Also returns
    ``logits`` [N, S-1, V] (unmasked) so callers can score a routing other than float64's own."""
    body = prefix + "transformer." + head_kind(sd, prefix) + "."
    h = hidden_states(sd, cfg, tokens, body)
    am = torch.as_tensor(tokens["attention_mask"])
    mask = am[:, 1:].unsqueeze(-1).double()
    logits = router_logits(sd, h[:, 1:], cfg["ln_eps"], prefix)
    full = torch.log1p(torch.relu(logits)) * mask
    w, ids = torch.topk(full, dim=2, k=topk)
    out = {"expert_repr": _linear(sd, h[:, 1:], prefix + "tok_project.") * mask, "expert_ids": ids,
           "expert_weights": w, "attention_mask": am[:, 1:].clone(), "logits": logits}
    if add_cls:
        out["cls_repr"] = _linear(sd, h[:, 0], prefix + "cls_project.")
    return out


def expert_score(q, d, q_ids, q_w, d_ids, d_w, pool="sum", q_cls=None, d_cls=None):
    """expert_sim_score (+ the CLS term) in float64: q [B, LQ, P], d [B, LD, P] (masked tokens already zero or given
    weight 0), ids [B, LQ, KQ] / [B, LD, KD] (2-D ids are COIL's KQ = KD = 1), weights of the same shape -> [B]."""
    if q_ids.dim() == 2:
        q_ids, d_ids, q_w, d_w = q_ids[..., None], d_ids[..., None], q_w[..., None], d_w[..., None]
    s = torch.bmm(q.double(), d.double().transpose(1, 2))                                  # B LQ LD
    match = q_ids[:, :, :, None, None] == d_ids[:, None, None, :, :]                        # B LQ KQ LD KD
    w = q_w.double()[:, :, :, None, None] * d_w.double()[:, None, None, :, :]
    e = s[:, :, None, :, None] * torch.where(match, w, torch.zeros((), dtype=w.dtype, device=w.device))
    B, LQ, KQ, LD, KD = e.shape
    m = e.reshape(B, LQ * KQ, LD * KD).max(-1).values
    if pool == "sum":
        out = m.sum(1)
    elif pool == "max":
        out = m.max(1).values
    else:
        raise NotImplementedError("Invalid query pooling! Available: [max, sum]")
    if q_cls is not None and d_cls is not None:
        out = out + (q_cls.double() * d_cls.double()).sum(1)
    return out
