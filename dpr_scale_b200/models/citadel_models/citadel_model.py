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

What runs: the body is ``dprb_encoder_fwd_tokens``; the head's dense layer + GELU is the library's GEMM with the
bias-GELU epilogue and its LayerNorm is ``dprb_ln_fwd`` (fp16 output); the decoder and its top-k are one
``dprb_search_topk`` call that never writes the logits: the tokens carry a 1 in column H and the decoder operand
[V, H + 8] (built once per weight version and cached) carries the bias there, so the fp32-accumulated inner product
is the logit.  Both operands are fp16 (11 significant bits against bf16's 8: fewer near-tied experts swap places).
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

ROUTER_DTYPE = torch.float16


class _TiedDecoder(nn.Module):
    """``decoder.{weight, bias}`` of the masked-LM head: the word embeddings and the head's bias under a second name, as
    HF ties them.  Saved under both names; on load the values come through the embedding / bias keys, and the decoder
    keys are only required to be present."""

    def __init__(self, owner):
        super().__init__()
        self.__dict__["_owner"] = owner

    def _save_to_state_dict(self, destination, prefix, keep_vars):
        for name, p in (("weight", self._owner.word_embeddings()), ("bias", self._owner.router_bias())):
            destination[prefix + name] = p if keep_vars else p.detach()

    def _load_from_state_dict(self, state_dict, prefix, local_metadata, strict, missing_keys, unexpected_keys,
                              error_msgs):
        for name in ("weight", "bias"):
            if strict and prefix + name not in state_dict:
                missing_keys.append(prefix + name)


class CITADELEncoder(nn.Module):
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
        H, V = cfg["hidden_size"], cfg["vocab_size"]
        if sd is None:
            body = HFEncoder(model_path="", dropout=dropout, _config=raw, _seed=_seed, _pooler=False)
        else:
            body = HFEncoder(model_path="", dropout=dropout, _config=raw, _state=sd, _pooler=False)
        self.config = cfg
        self.__dict__["_body"] = body   # not a submodule: its parameters are registered below, under the reference names
        self.__dict__["_router_cache"] = None
        self.bert_head = cfg["model_type"] == "bert"
        self.transformer = nn.Module()
        dense, norm = nn.Linear(H, H), nn.LayerNorm(H, eps=cfg["layer_norm_eps"])
        dense.weight.data.normal_(mean=0.0, std=cfg["initializer_range"])
        dense.bias.data.zero_()
        bias = nn.Parameter(torch.zeros(V))
        if self.bert_head:
            self.transformer.bert = body.transformer
            self.transformer.cls = nn.Module()
            head = self.transformer.cls.predictions = nn.Module()
            head.bias = bias
            head.transform = nn.Module()
            head.transform.dense, head.transform.LayerNorm = dense, norm
            names = {"dense": "cls.predictions.transform.dense.", "norm": "cls.predictions.transform.LayerNorm.",
                     "bias": "cls.predictions.bias"}
        else:
            self.transformer.roberta = body.transformer
            head = self.transformer.lm_head = nn.Module()
            head.dense, head.layer_norm = dense, norm
            head.bias = bias
            names = {"dense": "lm_head.dense.", "norm": "lm_head.layer_norm.", "bias": "lm_head.bias"}
        head.decoder = _TiedDecoder(self)
        self.__dict__["_head"] = head
        if sd is not None:                     # the masked-LM head of the checkpoint, when it has one (HF init if not)
            with torch.no_grad():
                for mod, key in ((dense, names["dense"]), (norm, names["norm"])):
                    if key + "weight" in sd:
                        mod.weight.copy_(sd[key + "weight"])
                        mod.bias.copy_(sd[key + "bias"])
                if names["bias"] in sd:
                    bias.copy_(sd[names["bias"]])
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

    def word_embeddings(self):
        return self._body.transformer.embeddings.word_embeddings.weight

    def router_bias(self):
        return self._head.bias

    def _head_layers(self):
        h = self._head
        return (h.transform.dense, h.transform.LayerNorm) if self.bert_head else (h.dense, h.layer_norm)

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

    def router_operand(self):
        """[V, H + 8] ROUTER_DTYPE: the decoder rows (the word embeddings) with the decoder bias in column H and zeros
        after it; rebuilt only when the weights change."""
        word, bias = self.word_embeddings(), self.router_bias()
        key = (word.data_ptr(), word._version, bias.data_ptr(), bias._version)
        cache = self._router_cache
        if cache is not None and cache[0] == key:
            return cache[1]
        V, H = word.shape
        op = torch.zeros(V, H + 8, dtype=ROUTER_DTYPE, device=word.device)
        op[:, :H] = word.detach()
        op[:, H] = bias.detach()
        self.__dict__["_router_cache"] = (key, op)
        return op

    def router_tokens(self, hidden):
        """[T, H + 8] ROUTER_DTYPE: the head's transform (dense + GELU on the GEMM epilogue, LayerNorm) of hidden bf16
        [T, H], with 1 in column H (it picks up the bias column of the operand) and zeros after it."""
        dense, norm = self._head_layers()
        T, H = hidden.shape
        w16 = torch.empty(H, H, dtype=torch.bfloat16, device=hidden.device)
        ops.cast_f32_bf16(dense.weight.detach().contiguous(), w16)
        act = ops.linear_fwd(hidden, w16, dense.bias.detach().contiguous(), ops.EPI_BIAS_GELU)
        y16 = torch.empty(T, H, dtype=torch.float16, device=hidden.device)
        ops.ln_fwd(act, norm.weight.detach().contiguous(), norm.bias.detach().contiguous(), norm.eps, y_res=y16)
        x = torch.zeros(T, H + 8, dtype=ROUTER_DTYPE, device=hidden.device)
        x[:, :H] = y16
        x[:, H] = 1.0
        return x

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
