"""float64 CPU restatement of the reference's SPLADE and dense (DPR) reranking paths:

  reps         dpr_scale/models/citadel_models/splade_model.py: logits = the masked-LM head (oracle.multivec.router_logits)
               on the last layer, then max over tokens 1.. of log(1 + relu(logits)) * attention_mask[:, 1:]
  pool         the dprb_splade_pool_fwd contract on compacted rows: out[n, v] = log1p(relu(max over rows off[n] ..
               off[n+1] - 1 of x[:, :K] . W[v, :K] + bias[v])), 0 for an empty range
  dense        HFEncoder.forward: the CLS vector of the last layer, through the optional Linear + LayerNorm projection
  rerank_score dpr_scale/task/dpr_rerank_task.py _eval_step: sum(q_repr * ctx_repr, 1)
The encoder layers are oracle.encoder's.  ``sd`` holds an encoder's state_dict keys under ``prefix``.
"""
import torch

from .colbert import _double, hidden_states
from .encoder import encode
from .multivec import head_kind, router_logits


def reps(sd, cfg, tokens, prefix=""):
    """SPLADEEncoder.forward(tokens) in float64 [N, V]."""
    body = prefix + "transformer." + head_kind(sd, prefix) + "."
    h = hidden_states(sd, cfg, tokens, body)
    mask = torch.as_tensor(tokens["attention_mask"])[:, 1:].unsqueeze(-1).double()
    logits = router_logits(sd, h[:, 1:], cfg["ln_eps"], prefix)
    return (torch.log1p(torch.relu(logits)) * mask).max(1).values


def pool(x, W, off, K, bias=None):
    """The dprb_splade_pool_fwd contract in float64 (x [T, >= K], W [V, >= K], off [N + 1], bias [V] or None)."""
    x, W = x[:, :K].double(), W[:, :K].double()
    off = [int(o) for o in torch.as_tensor(off).tolist()]
    out = torch.zeros(len(off) - 1, W.shape[0], dtype=torch.float64, device=W.device)
    for n in range(len(off) - 1):
        if off[n + 1] > off[n]:
            m = (x[off[n]:off[n + 1]] @ W.T).max(0).values
            if bias is not None:
                m = m + bias.double()
            out[n] = torch.log1p(torch.relu(m))
    return out


def dense(sd, cfg, tokens, prefix=""):
    """HFEncoder.forward(tokens) in float64 [N, H or P]."""
    return encode(_double(sd), cfg, {k: torch.as_tensor(v) for k, v in tokens.items()}, prefix + "transformer.")


def rerank_score(q, d):
    return (q.double() * d.double()).sum(1)
