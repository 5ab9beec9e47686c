"""CITADELEncoder — drop-in for ``dpr_scale.models.citadel_models.citadel_model.CITADELEncoder`` (the reference's
dpr_scale/models/citadel_models/citadel_model.py:12-82): each token is routed through the masked-LM head to its top-k
vocabulary "experts", forward only.

Same constructor (``model_path, dropout, tok_projection_dim, cls_projection_dim``) and ``state_dict`` keys and shapes as
the reference's ``transformer = AutoModelForMaskedLM(...)`` plus ``cls_project.0.*`` / ``tok_project.0.*``:
``transformer.bert.*`` (no pooler) and ``transformer.cls.predictions.{bias, transform.dense.*, transform.LayerNorm.*,
decoder.weight, decoder.bias}`` for BERT, ``transformer.roberta.*`` and ``transformer.lm_head.{bias, dense.*,
layer_norm.*, decoder.weight, decoder.bias}`` for RoBERTa / XLM-R.  As in HF, the decoder is tied: its weight IS the
word-embedding table and its bias IS the head's bias, so both appear under two names and load through the body / head
keys.  Reference checkpoints load strictly.

``forward(tokens, topk=1, add_cls=False)`` returns the reference's ``expert_repr`` (fp32, masked), ``expert_ids``
(int64), ``expert_weights`` = log(1 + relu(logit)) of the chosen experts (0 on masked tokens), ``attention_mask`` and,
with ``add_cls``, ``cls_repr``.  The training statistics (``router_repr``, ``router_mask``, ``router_softmax_repr``,
``avg_*_num_experts``) need the full [tokens, vocab] logits, which this path never materialises: they are not returned.
Masked tokens get weight 0; their ids are unspecified.  Where fewer than k logits are positive the extra experts have
weight 0, as in the reference, and which ids they carry does not change any score.

What runs: the body is ``dprb_encoder_fwd_tokens``; the head's transform and the cached decoder operand are the shared
masked-LM head (mlm_head.py); the decoder and its top-k are one ``dprb_search_topk`` call that never writes the
logits.  Both operands are fp16 (11 significant bits against bf16's 8: fewer near-tied experts swap places).
"""
import json
import os
from typing import Optional

import torch
import torch.nn as nn

from ... import ops
from ..hf_model import HFEncoder, ParamLayout, _normalise_config
from .coil_model import cls_reps
from .colbert_model import _KINDS, encode_tokens, linear_bf16
from .mlm_head import MaskedLMHeadMixin

class CITADELEncoder(MaskedLMHeadMixin, nn.Module):
    def __init__(self, model_path: str = "bert-base-uncased", dropout: float = 0.1,
                 tok_projection_dim: Optional[int] = None, cls_projection_dim: Optional[int] = None, _config=None,
                 _seed: int = 0):
        super().__init__()
        if _config is not None:
            raw, sd = dict(_config), None
        else:
            if not os.path.isdir(model_path):
                raise FileNotFoundError(f"model_path {model_path!r} is not a local directory "
                                        "(no network here: hub names cannot be resolved)")
            with open(os.path.join(model_path, "config.json")) as f:
                raw = json.load(f)
            self._check_config(raw, tok_projection_dim, cls_projection_dim)      # fail before reading the weights
            _, sd = HFEncoder._read_pretrained(model_path)
        cfg = self._check_config(raw, tok_projection_dim, cls_projection_dim)
        H = cfg["hidden_size"]
        if sd is None:
            body = HFEncoder(model_path="", dropout=dropout, _config=raw, _seed=_seed, _pooler=False)
        else:
            body = HFEncoder(model_path="", dropout=dropout, _config=raw, _state=sd, _pooler=False)
        self.config = cfg
        self.__dict__["_body"] = body   # not a submodule: its parameters are registered below, under the reference names
        self._build_head(body, cfg, sd)
        self.cls_project = nn.Identity()
        if cls_projection_dim:
            linear = nn.Linear(H, cls_projection_dim)
            linear.weight.data.normal_(mean=0.0, std=0.02)
            self.cls_project = nn.Sequential(linear)
        self.tok_project = nn.Identity()
        if tok_projection_dim:
            linear = nn.Linear(H, tok_projection_dim)
            linear.weight.data.normal_(mean=0.0, std=0.02)
            self.tok_project = nn.Sequential(linear)
        self.eval()

    @staticmethod
    def _check_config(raw, tok_projection_dim, cls_projection_dim):
        """Normalised config; ValueError for what the kernels cannot run, before any GPU work."""
        kind = raw.get("model_type", "bert")
        if kind not in _KINDS:
            raise ValueError(f"CITADELEncoder supports BERT, RoBERTa and XLM-R encoders (model_type={kind!r})")
        cfg = _normalise_config(raw)
        ParamLayout(cfg)                  # head_dim 64, H / I multiples of 8, H <= 1024
        H = cfg["hidden_size"]
        ops.maxsim_expert_check(2, 2, int(tok_projection_dim) if tok_projection_dim else H, 1, 1,
                                int(cls_projection_dim) if cls_projection_dim else H)
        return cfg

    @classmethod
    def from_config(cls, config, tok_projection_dim: Optional[int] = None, cls_projection_dim: Optional[int] = None,
                    seed: int = 0):
        """Random init (HF scheme) from a config dict, without a checkpoint directory."""
        return cls(model_path="", dropout=0.0, tok_projection_dim=tok_projection_dim,
                   cls_projection_dim=cls_projection_dim, _config=dict(config), _seed=seed)

    # ------------------------------------------------------------------ forward
    def _check_call(self, tokens, topk):
        if torch.is_grad_enabled():
            raise ValueError("CITADELEncoder runs forward only (training is not implemented): call it under "
                             "torch.no_grad()")
        S = tokens["input_ids"].shape[-1]
        if not 2 <= S <= ops.MAXSIM_MAX_S:
            raise ValueError(f"CITADELEncoder needs 2 .. {ops.MAXSIM_MAX_S} tokens per sequence (got {S}): token 0 "
                             "is dropped")
        if not 1 <= int(topk) <= min(ops.MAXSIM_MAX_EXPERTS, self.config["vocab_size"]):
            raise ValueError(f"CITADELEncoder routes each token to 1 .. {ops.MAXSIM_MAX_EXPERTS} experts (got "
                             f"topk={topk})")

    def route(self, hidden, topk):
        """(logits fp32 [T, k] descending, ids int64 [T, k]) of the top-k experts of every row of hidden bf16 [T, H]."""
        return ops.search_topk(self.router_tokens(hidden), self.router_operand(), int(topk))

    def expert_reps(self, tokens, topk=1, add_cls=False):
        """(reps bf16 [N, S, P], ids int32 [N, S, k], weights fp32 [N, S, k], cls bf16 [N, Pc] or None): every token
        with token 0, unmasked reps; the weights are log1p(relu(logit)) of the chosen experts, 0 on masked tokens."""
        self._check_call(tokens, topk)
        hidden, am, N, S = encode_tokens(self._body, tokens)
        logit, ids = self.route(hidden, topk)
        w = torch.log1p(torch.relu(logit)) * am.view(N * S, 1)
        reps = hidden if isinstance(self.tok_project, nn.Identity) else linear_bf16(self.tok_project[0], hidden)
        cls = cls_reps(self.cls_project, hidden, N, S) if add_cls else None
        k = int(topk)
        return reps.view(N, S, -1), ids.to(torch.int32).view(N, S, k), w.view(N, S, k), cls

    def forward(self, tokens, topk=1, add_cls=False):
        reps, ids, w, cls = self.expert_reps(tokens, topk, add_cls)
        am = torch.as_tensor(tokens["attention_mask"]).to(reps.device)
        keep = am[:, 1:].unsqueeze(-1) != 0
        ret = {"attention_mask": am[:, 1:].clone()}
        if add_cls:
            ret["cls_repr"] = cls.float()
        ret["expert_ids"] = ids[:, 1:].long()
        ret["expert_repr"] = torch.where(keep, reps[:, 1:, :].float(), torch.zeros((), device=reps.device))
        ret["expert_weights"] = w[:, 1:].contiguous()
        return ret
