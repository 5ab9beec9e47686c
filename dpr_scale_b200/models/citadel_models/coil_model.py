"""COILEncoder — drop-in for ``dpr_scale.models.citadel_models.coil_model.COILEncoder`` (the reference's
dpr_scale/models/citadel_models/coil_model.py:12-61): ColBERT plus exact lexical matching, and optionally a CLS vector,
forward only.

Same constructor (``model_path, dropout, projection_dim, cls_projection_dim``), same call (``forward(tokens,
add_cls=False) -> {"expert_repr", "expert_ids", "expert_weights", "attention_mask"[, "cls_repr"]}``: the projected last
layer without token 0 times ``attention_mask[:, 1:]`` in fp32, ``input_ids[:, 1:]`` as the expert ids, the mask as the
weights, and ``cls_project(hidden_states[-1][:, 0])`` with ``add_cls``), same ``state_dict`` keys and shapes as the
reference (``transformer.*`` with the pooler, ``project.0.*``, ``cls_project.0.*``), so reference checkpoints load
strictly.

The body and token projection are ColBERTEncoder's (``dprb_encoder_fwd_tokens`` and the library's GEMM); the CLS
projection is the same GEMM on the token-0 rows.  ``expert_reps`` returns what ``dprb_maxsim_expert_fwd`` reads: the
unmasked projected tokens, the ids and weights (the mask) of every token and the bf16 CLS vectors.  Training is not
implemented: a forward with gradients enabled raises ValueError before any GPU work.
"""
from typing import Optional

import torch
import torch.nn as nn

from ... import ops
from .colbert_model import ColBERTEncoder, linear_bf16


def cls_reps(project, hidden, N, S):
    """bf16 [N, Pc]: ``project`` (a Sequential(Linear) or the identity) of the token-0 rows of hidden bf16 [N*S, H]."""
    h0 = hidden.view(N, S, -1)[:, 0].contiguous()
    return h0 if isinstance(project, nn.Identity) else linear_bf16(project[0], h0)


class COILEncoder(ColBERTEncoder):
    def __init__(self, model_path: str = "roberta-base", dropout: float = 0.1, projection_dim: Optional[int] = None,
                 cls_projection_dim: Optional[int] = None, _config=None, _seed: int = 0):
        if cls_projection_dim:
            ops.maxsim_expert_check(2, 2, 8, 1, 1, int(cls_projection_dim))     # fail before reading the weights
        super().__init__(model_path=model_path, dropout=dropout, projection_dim=projection_dim, _config=_config,
                         _seed=_seed)
        self.cls_project = nn.Identity()
        if cls_projection_dim:
            linear = nn.Linear(self.config["hidden_size"], cls_projection_dim)
            linear.weight.data.normal_(mean=0.0, std=0.02)
            self.cls_project = nn.Sequential(linear)
        self.eval()

    @classmethod
    def from_config(cls, config, projection_dim: Optional[int] = None, cls_projection_dim: Optional[int] = None,
                    seed: int = 0):
        """Random init (HF scheme) from a config dict, without a checkpoint directory."""
        return cls(model_path="", dropout=0.0, projection_dim=projection_dim, cls_projection_dim=cls_projection_dim,
                   _config=dict(config), _seed=seed)

    def expert_reps(self, tokens, add_cls=False, **kwargs):
        """(reps bf16 [N, S, P], ids int32 [N, S, 1], weights fp32 [N, S, 1], cls bf16 [N, Pc] or None): every token
        with token 0, unmasked; the weights are the attention mask, so padded tokens score 0."""
        hidden, am, N, S = self._hidden(tokens)
        reps = hidden if isinstance(self.project, nn.Identity) else linear_bf16(self.project[0], hidden)
        ids = torch.as_tensor(tokens["input_ids"]).to(am.device, torch.int32).view(N, S, 1)
        cls = cls_reps(self.cls_project, hidden, N, S) if add_cls else None
        return reps.view(N, S, -1), ids, am.float().view(N, S, 1), cls

    def forward(self, tokens, add_cls=False, **kwargs):
        reps, ids, w, cls = self.expert_reps(tokens, add_cls)
        am = torch.as_tensor(tokens["attention_mask"]).to(reps.device)
        keep = am[:, 1:].unsqueeze(-1) != 0
        ret = {}
        if add_cls:
            ret["cls_repr"] = cls.float()
        ret["expert_repr"] = torch.where(keep, reps[:, 1:, :].float(), torch.zeros((), device=reps.device))
        ret["expert_ids"] = torch.as_tensor(tokens["input_ids"]).to(reps.device)[:, 1:].clone()
        ret["expert_weights"] = am[:, 1:].clone()
        ret["attention_mask"] = am[:, 1:].clone()
        return ret
