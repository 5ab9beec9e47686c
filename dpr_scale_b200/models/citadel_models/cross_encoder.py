"""CrossEncoder — drop-in for ``dpr_scale.models.citadel_models.cross_encoder.CrossEncoder``
(/root/reference/dpr_scale/models/citadel_models/cross_encoder.py:11-26): a BERT or RoBERTa / XLM-R
``...ForSequenceClassification`` checkpoint scoring ``[CLS] query [SEP] passage [SEP]`` pairs, and its training with a
grouped softmax cross-entropy (``group_ce``), which the reference does not implement.

Same constructor (``model_path``), same call (``forward(tokens) -> logits fp32 [N, num_labels]`` under ``no_grad``), same
``state_dict`` keys and shapes as the reference's ``self.transformer = AutoModelForSequenceClassification(...)``:
  BERT:            ``transformer.bert.*`` (pooler included) + ``transformer.classifier.{weight,bias}``;
  RoBERTa / XLM-R: ``transformer.roberta.*`` (no pooler) + ``transformer.classifier.{dense,out_proj}.{weight,bias}``,
so reference checkpoints load strictly.

What runs: the encoder body is HFEncoder's forward-only mode (flat fp32 arena, bf16 shadow, CLS-pruned last layer: only
token 0 of the last layer is computed, which is all the head reads).  The head is the library's GEMM for its dense layer
(fp32 output) and ``dprb_seqcls_head_fwd`` for tanh, the label projection and the label max.  Dropout is the identity:
the reference runs the model in eval mode.

Training (``group_ce`` in train mode with grad enabled, one label): the body runs HFEncoder's training forward with
``hidden_dropout_prob``; RoBERTa's head drops its CLS rows (site 5) before the dense GEMM; ``dprb_seqcls_group_ce`` takes
tanh, the head's dropout (site 4; p = ``classifier_dropout``, else ``hidden_dropout_prob``), the label projection, the
grouped cross-entropy and the head's backward down to the dense layer's output gradient in one pass; the library's GEMM
then gives the dense layer's weight gradient and the CLS rows' gradient, which HFEncoder's backward takes.  Both head
sites are keyed by the body forward's dropout seed (``dprb_dropout_mask`` replays them).

``num_labels=n`` loads like HF's ``from_pretrained(path, num_labels=n)``: a head tensor the checkpoint lacks, or holds
with another shape, keeps its fresh HF-scheme initialisation (seeded), so training can start from a plain BERT or
RoBERTa checkpoint.  With ``num_labels=None`` the checkpoint's head is required (``KeyError`` when missing).
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


def _check_config(raw_cfg: Mapping, num_labels=None):
    """(normalised config, body name, num_labels); ValueError for what the kernels cannot run, before any GPU work."""
    if num_labels is not None:
        raw_cfg = {k: v for k, v in raw_cfg.items() if k != "id2label"}
        raw_cfg["num_labels"] = int(num_labels)
    kind = raw_cfg.get("model_type", "bert")
    if kind not in _BODY:
        raise ValueError(f"CrossEncoder supports BERT, RoBERTa and XLM-R sequence classifiers (model_type={kind!r})")
    cfg = _normalise_config(raw_cfg)
    ParamLayout(cfg)                  # head_dim 64, H / I multiples of 8, H <= 1024
    L = num_labels_of(raw_cfg)
    if not 1 <= L <= ops.SEQCLS_MAX_LABELS:
        raise ValueError(f"CrossEncoder head supports 1 .. {ops.SEQCLS_MAX_LABELS} labels (num_labels={L})")
    return cfg, _BODY[kind], L


class _GroupCE(torch.autograd.Function):
    """(loss, logits) of the grouped cross-entropy from the body's CLS rows; the head's backward was computed by the
    forward's kernel, so backward runs the dense layer's two GEMMs and its bias column sums."""

    @staticmethod
    def forward(ctx, cls, w_dense, b_dense, w_out, b_out, labels, G, p_head, p_in, seed):
        N, H = cls.shape
        dev = cls.device
        drop_in = None
        if p_in > 0:
            drop_in = ops.dropout_mask(N, H, p_in, seed, 0, ops.DROP_SITE_HEAD_IN).float().mul_(_keep_scale(p_in))
            cls = cls * drop_in
        x16 = torch.empty(N, H, dtype=torch.bfloat16, device=dev)
        w16 = torch.empty(H, H, dtype=torch.bfloat16, device=dev)
        ops.cast_f32_bf16(cls.contiguous(), x16)
        ops.cast_f32_bf16(w_dense.detach().contiguous(), w16)
        pre = torch.empty(N, H, dtype=torch.float32, device=dev)
        ops.gemm(x16, w16, pre, N, H, H, H, H, H, False, False, ops.EPI_F32_STORE, b_dense.detach().contiguous())
        loss, logits, dpre, dw_out, db_out = ops.seqcls_group_ce(pre, w_out.detach(), b_out.detach().contiguous(),
                                                                 labels, G, p_head, seed)
        ctx.save_for_backward(x16, w16, dpre, dw_out, db_out, drop_in)
        ctx.mark_non_differentiable(logits)
        return loss.view(()), logits

    @staticmethod
    def backward(ctx, g, _):
        x16, w16, dpre, dw_out, db_out, drop_in = ctx.saved_tensors
        N, H = x16.shape
        dev = x16.device
        dw = torch.zeros(H, H, dtype=torch.float32, device=dev)
        ops.gemm(dpre, x16, dw, H, H, N, H, H, H, True, True, ops.EPI_F32_ATOMIC_ADD, None, splits=0)
        db = torch.zeros(H, dtype=torch.float32, device=dev)
        ops.colsum(dpre, db)
        dx = torch.empty(N, H, dtype=torch.float32, device=dev)
        ops.gemm(dpre, w16, dx, N, H, H, H, H, H, False, True, ops.EPI_F32_STORE, None)
        if drop_in is not None:
            dx.mul_(drop_in)
        g = g.float()
        # dw_out / db_out are saved: scale copies, so a second backward (retain_graph=True) sees them unscaled
        return (dx.mul_(g), dw.mul_(g), db.mul_(g), dw_out * g, db_out * g, None, None, None, None, None)


def _keep_scale(p):
    """The kernels' multiplier of a kept element: p is quantised to 16 bits (include/dprb.h, dropout sites)."""
    t = min(int(float(torch.tensor(p, dtype=torch.float32)) * 65536.0 + 0.5), 65535)
    return 1.0 / (1.0 - t / 65536.0) if t else 1.0


class CrossEncoder(nn.Module):
    def __init__(self, model_path: str = "cross-encoder/ms-marco-MiniLM-L-6-v2", _config=None, _seed: int = 0,
                 num_labels=None):
        super().__init__()
        if _config is not None:
            raw, sd = dict(_config), None
        else:
            if not os.path.isdir(model_path):
                raise FileNotFoundError(f"model_path {model_path!r} is not a local directory "
                                        "(no network here: hub names cannot be resolved)")
            with open(os.path.join(model_path, "config.json")) as f:
                raw = json.load(f)
            _check_config(raw, num_labels)        # fail before reading the weights
            _, sd = HFEncoder._read_pretrained(model_path)
        cfg, body_name, L = _check_config(raw, num_labels)
        H = cfg["hidden_size"]
        is_bert = body_name == "bert"
        if sd is None:
            body = HFEncoder(model_path="", dropout=0.0, _config=raw, _seed=_seed, _pooler=is_bert)
        else:
            body = HFEncoder(model_path="", dropout=0.0, _config=raw, _state=sd, _pooler=is_bert)
        body.eval()
        self.config, self.num_labels, self.body_name = cfg, L, body_name
        # dropout of training (HF's config fields; the body kernels take one p for hidden and attention dropout)
        self.hidden_dropout = float(raw.get("hidden_dropout_prob", 0.1))
        self.attention_dropout = float(raw.get("attention_probs_dropout_prob", 0.1))
        cd = raw.get("classifier_dropout")
        self.head_dropout = self.hidden_dropout if cd is None else float(cd)
        body.dropout = self.hidden_dropout
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
            self._load_head(sd, fresh_ok=num_labels is not None)
        self.eval()

    @classmethod
    def from_config(cls, config: Mapping, seed: int = 0, num_labels=None):
        """Random init (HF scheme) from a config dict, without a checkpoint directory."""
        return cls(model_path="", _config=dict(config), _seed=seed, num_labels=num_labels)

    def train(self, mode: bool = True):
        super().train(mode)
        self._body.train(mode)      # the body is not a submodule: its mode selects the training forward
        return self

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

    def _load_head(self, sd, fresh_ok=False):
        """The head tensors of an HF ``...ForSequenceClassification`` state dict (the body was loaded by HFEncoder).
        fresh_ok: a missing or differently shaped tensor keeps its initialisation (HF's from_pretrained(num_labels=n))."""
        pre = self.body_name + "."
        names = {"bert": ["bert.pooler.dense", "classifier"],
                 "roberta": ["classifier.dense", "classifier.out_proj"]}[self.body_name]
        for lin, name in zip(self._head_linears(), names):
            for p in ("weight", "bias"):
                key = next((k for k in (name + "." + p, name.replace(pre, "", 1) + "." + p) if k in sd), None)
                if fresh_ok and (key is None or tuple(sd[key].shape) != tuple(getattr(lin, p).shape)):
                    continue
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

    def check_training(self, rows, group_size):
        """ValueError, before any GPU work, for what group_ce cannot train: more than one label, groups that are not
        whole or outside 2 .. ops.SEQCLS_GROUP_MAX, or attention and hidden dropout probabilities that differ."""
        if self.num_labels != 1:
            raise ValueError(f"cross-encoder training needs one relevance label (num_labels={self.num_labels}); "
                             "give num_labels=1")
        ops.seqcls_group_ce_check(rows, self.config["hidden_size"], int(group_size))
        if self.attention_dropout != self.hidden_dropout:
            raise ValueError(f"attention_probs_dropout_prob={self.attention_dropout} differs from hidden_dropout_prob="
                             f"{self.hidden_dropout}: the encoder kernels take one dropout probability")

    def group_ce(self, tokens, labels, group_size):
        """(loss, logits fp32 [N]) of groups of ``group_size`` consecutive pairs, ``labels`` int64 [N / group_size]
        naming each group's relevant pair: the mean over groups of the softmax cross-entropy.  In train mode with grad
        enabled the loss is differentiable and dropout is on; otherwise nothing is saved and dropout is off."""
        N = tokens["input_ids"].shape[0]
        self.check_training(N, group_size)
        dense, out = self._head_linears()
        body = self._body
        if self.training and torch.is_grad_enabled():
            cls = body(tokens)                                   # HFEncoder's training forward, fp32 [N, H]
            seed = body.last_dropout[1]
            p_head, p_in = self.head_dropout, (self.head_dropout if self.body_name == "roberta" else 0.0)
        else:
            with torch.no_grad():
                cls, _ = body._run_forward(tokens, False)
            seed, p_head, p_in = 0, 0.0, 0.0
        labels = torch.as_tensor(labels).to(cls.device, torch.int64)
        return _GroupCE.apply(cls, dense.weight, dense.bias, out.weight, out.bias, labels, int(group_size), p_head,
                              p_in, seed)
