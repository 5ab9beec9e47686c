"""CrossEncoder — drop-in for ``dpr_scale.models.citadel_models.cross_encoder.CrossEncoder``
(/root/reference/dpr_scale/models/citadel_models/cross_encoder.py:11-26): a BERT or RoBERTa / XLM-R
``...ForSequenceClassification`` checkpoint scoring ``[CLS] query [SEP] passage [SEP]`` pairs, forward only.

Same constructor (``model_path``), same call (``forward(tokens) -> logits fp32 [N, num_labels]`` under ``no_grad``), same
``state_dict`` keys and shapes as the reference's ``self.transformer = AutoModelForSequenceClassification(...)``:
  BERT:            ``transformer.bert.*`` (pooler included) + ``transformer.classifier.{weight,bias}``;
  RoBERTa / XLM-R: ``transformer.roberta.*`` (no pooler) + ``transformer.classifier.{dense,out_proj}.{weight,bias}``,
so reference checkpoints load strictly.

What runs: the encoder body is HFEncoder's forward-only mode (flat fp32 arena, bf16 shadow, CLS-pruned last layer: only
token 0 of the last layer is computed, which is all the head reads).  The head is the library's GEMM for its dense layer
(fp32 output) and ``dprb_seqcls_head_fwd`` for tanh, the label projection and the label max.  Dropout is the identity:
the reference runs the model in eval mode.
"""
import json
import os
from typing import Mapping

import torch
import torch.nn as nn

from ... import ops
from ..hf_model import HFEncoder, ParamLayout, _normalise_config

_BODY = {"bert": "bert", "roberta": "roberta", "xlm-roberta": "roberta"}


def num_labels_of(raw_cfg: Mapping) -> int:
    """PretrainedConfig's rule: the length of ``id2label`` when the config has one, else ``num_labels`` (default 2)."""
    if raw_cfg.get("id2label") is not None:
        return len(raw_cfg["id2label"])
    return int(raw_cfg.get("num_labels", 2))


def _check_config(raw_cfg: Mapping):
    """(normalised config, body name, num_labels); ValueError for what the kernels cannot run, before any GPU work."""
    kind = raw_cfg.get("model_type", "bert")
    if kind not in _BODY:
        raise ValueError(f"CrossEncoder supports BERT, RoBERTa and XLM-R sequence classifiers (model_type={kind!r})")
    cfg = _normalise_config(raw_cfg)
    ParamLayout(cfg)                  # head_dim 64, H / I multiples of 8, H <= 1024
    L = num_labels_of(raw_cfg)
    if not 1 <= L <= ops.SEQCLS_MAX_LABELS:
        raise ValueError(f"CrossEncoder head supports 1 .. {ops.SEQCLS_MAX_LABELS} labels (num_labels={L})")
    return cfg, _BODY[kind], L


class CrossEncoder(nn.Module):
    def __init__(self, model_path: str = "cross-encoder/ms-marco-MiniLM-L-6-v2", _config=None, _seed: int = 0):
        super().__init__()
        if _config is not None:
            raw, sd = dict(_config), None
        else:
            if not os.path.isdir(model_path):
                raise FileNotFoundError(f"model_path {model_path!r} is not a local directory "
                                        "(no network here: hub names cannot be resolved)")
            with open(os.path.join(model_path, "config.json")) as f:
                raw = json.load(f)
            _check_config(raw)        # fail before reading the weights
            _, sd = HFEncoder._read_pretrained(model_path)
        cfg, body_name, L = _check_config(raw)
        H = cfg["hidden_size"]
        is_bert = body_name == "bert"
        if sd is None:
            body = HFEncoder(model_path="", dropout=0.0, _config=raw, _seed=_seed, _pooler=is_bert)
        else:
            body = HFEncoder(model_path="", dropout=0.0, _config=raw, _state=sd, _pooler=is_bert)
        body.eval()
        self.config, self.num_labels, self.body_name = cfg, L, body_name
        self.__dict__["_body"] = body  # not a submodule: its parameters are registered below, under the HF names
        self.transformer = nn.Module()
        self.transformer.add_module(body_name, body.transformer)
        if is_bert:
            self.transformer.add_module("classifier", nn.Linear(H, L))
        else:
            head = nn.Module()
            head.add_module("dense", nn.Linear(H, H))
            head.add_module("out_proj", nn.Linear(H, L))
            self.transformer.add_module("classifier", head)
        self._init_head(cfg, _seed)
        if sd is not None:
            self._load_head(sd)
        self.eval()

    @classmethod
    def from_config(cls, config: Mapping, seed: int = 0):
        """Random init (HF scheme) from a config dict, without a checkpoint directory."""
        return cls(model_path="", _config=dict(config), _seed=seed)

    # ------------------------------------------------------------------ head parameters
    def _head_linears(self):
        """(dense, out): the head's dense layer (BERT pooler / RoBERTa classifier.dense) and its label projection."""
        t = self.transformer
        if self.body_name == "bert":
            return t.bert.pooler.dense, t.classifier
        return t.classifier.dense, t.classifier.out_proj

    def _init_head(self, cfg, seed):
        g = torch.Generator().manual_seed(seed + 1)
        with torch.no_grad():
            for lin in self._head_linears():
                lin.weight.normal_(0.0, cfg["initializer_range"], generator=g)
                lin.bias.zero_()

    def _load_head(self, sd):
        """The head tensors of an HF ``...ForSequenceClassification`` state dict (the body was loaded by HFEncoder)."""
        pre = self.body_name + "."
        names = {"bert": ["bert.pooler.dense", "classifier"],
                 "roberta": ["classifier.dense", "classifier.out_proj"]}[self.body_name]
        for lin, name in zip(self._head_linears(), names):
            for p in ("weight", "bias"):
                key = next((k for k in (name + "." + p, name.replace(pre, "", 1) + "." + p) if k in sd), None)
                if key is None:
                    raise KeyError(f"checkpoint is missing the classification head tensor {name}.{p}")
                if tuple(sd[key].shape) != tuple(getattr(lin, p).shape):
                    raise ValueError(f"{key}: shape {tuple(sd[key].shape)} != {tuple(getattr(lin, p).shape)}")
                with torch.no_grad():
                    getattr(lin, p).copy_(sd[key])

    # ------------------------------------------------------------------ forward
    def logits_and_scores(self, tokens):
        """(logits fp32 [N, num_labels], score fp32 [N] = max over labels) of a batch of pair tokens."""
        with torch.no_grad():
            cls, _ = self._body._run_forward(tokens, False)          # last-layer token 0, fp32 [N, H]
            dense, out = self._head_linears()
            N, H = cls.shape
            dev = cls.device
            x16 = torch.empty(N, H, dtype=torch.bfloat16, device=dev)
            w16 = torch.empty(H, H, dtype=torch.bfloat16, device=dev)
            ops.cast_f32_bf16(cls, x16)
            ops.cast_f32_bf16(dense.weight.detach().contiguous(), w16)
            pre = torch.empty(N, H, dtype=torch.float32, device=dev)
            ops.gemm(x16, w16, pre, N, H, H, H, H, H, False, False, ops.EPI_F32_STORE, dense.bias.detach().contiguous())
            return ops.seqcls_head_fwd(pre, out.weight.detach().contiguous(), out.bias.detach().contiguous())

    def forward(self, tokens):
        return self.logits_and_scores(tokens)[0]
