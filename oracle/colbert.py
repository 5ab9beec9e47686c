"""float64 CPU restatement of the reference's ColBERT reranking path:

  expert_repr  dpr_scale/models/citadel_models/colbert_model.py:39-44: hidden_states[-1][:, 1:, :] -> project
               (Linear, or the identity) -> * attention_mask[:, 1:]
  maxsim       dpr_scale/task/citadel_eval_task.py:236-265 (expert_sim_score without expert ids): bmm(q, d^T), max over
               the passage tokens, then sum (query_pool="sum") or max ("max") over the query tokens
The encoder layers are oracle.encoder's.  ``sd`` holds a ColBERTEncoder's state_dict keys (``transformer.*`` +
optional ``project.0.{weight,bias}``) under ``prefix``.
"""
import torch

from .encoder import embeddings, layer, roberta_position_ids


def _double(sd):
    return {k: torch.as_tensor(v).double() if torch.as_tensor(v).is_floating_point() else torch.as_tensor(v)
            for k, v in sd.items()}


def hidden_states(sd, cfg, tokens, prefix="transformer."):
    """Last-layer output of every token, float64 [N, S, H] (cfg: oracle.encoder keys layers, heads, ln_eps, pad_id,
    roberta)."""
    sd = _double(sd)
    tokens = {k: torch.as_tensor(v) for k, v in tokens.items()}
    ids = tokens["input_ids"]
    N, S = ids.shape
    tt = tokens.get("token_type_ids")
    tt = torch.zeros_like(ids) if tt is None else tt
    am = tokens.get("attention_mask")
    pos = roberta_position_ids(ids, cfg["pad_id"]) if cfg.get("roberta", False) else \
        torch.arange(S).unsqueeze(0).expand(N, S)
    x = embeddings(sd, prefix, ids, tt, pos, cfg["ln_eps"])
    for l in range(cfg["layers"]):
        x = layer(x, sd, f"{prefix}encoder.layer.{l}.", cfg["heads"], am, cfg["ln_eps"])
    return x


def project(sd, x, prefix="project."):
    """The optional Linear of ColBERTEncoder.project (identity without one)."""
    if prefix + "0.weight" not in sd:
        return x
    w = torch.as_tensor(sd[prefix + "0.weight"]).double()
    b = torch.as_tensor(sd[prefix + "0.bias"]).double()
    return x @ w.T + b


def expert_repr(sd, cfg, tokens, prefix=""):
    """ColBERTEncoder.forward(tokens)["expert_repr"] in float64 [N, S-1, P]."""
    h = hidden_states(sd, cfg, tokens, prefix + "transformer.")
    am = torch.as_tensor(tokens["attention_mask"])
    return project(sd, h[:, 1:, :], prefix + "project.") * am[:, 1:].unsqueeze(-1).double()


def maxsim(q, d, pool="sum"):
    """expert_sim_score: q [B, LQ, P], d [B, LD, P] (already masked: padded tokens are zero vectors) -> [B]."""
    s = torch.bmm(q.double(), d.double().transpose(1, 2))
    m = s.max(-1).values
    if pool == "sum":
        return m.sum(1)
    if pool == "max":
        return m.max(1).values
    raise NotImplementedError("Invalid query pooling! Available: [max, sum]")


def maxsim_tokens(q, d, q_mask, d_mask, q_index, pool="sum"):
    """The dprb_maxsim_fwd contract in float64: unmasked tokens with token 0 [nq, SQ, P] / [B, SD, P], their masks and
    the query row of each pair; masked tokens become zero vectors as in the reference."""
    q = q.double() * torch.as_tensor(q_mask).double().unsqueeze(-1)
    d = d.double() * torch.as_tensor(d_mask).double().unsqueeze(-1)
    return maxsim(q[torch.as_tensor(q_index).long(), 1:], d[:, 1:], pool)
