"""SPLADEEncoder — drop-in for ``dpr_scale.models.citadel_models.splade_model.SPLADEEncoder``: a BERT or RoBERTa
masked-LM encoder whose representation is a vocabulary-sized vector, forward only.

Same constructor (``model_path, dropout``), same call (``forward(tokens) -> fp32 [N, V]`` = the max over tokens 1.. of
log(1 + relu(logits)) * attention_mask) and the same ``state_dict`` keys and shapes as the reference's ``transformer =
AutoModelForMaskedLM(...)``: those of the shared masked-LM head (mlm_head.py), the decoder tied to the word embeddings
and the head bias.  Reference checkpoints load strictly.

What runs: the body is ``dprb_encoder_fwd_tokens``; the valid tokens (token 0 and masked tokens dropped) are compacted
into contiguous rows per sequence, so neither the head nor the decoder computes padding; the head's transform and the
cached fp16 decoder operand are the shared masked-LM head's; ``dprb_splade_pool_fwd`` runs the decoder GEMM with the
max-pool in its epilogue (the [tokens, V] logits are never written) and adds the head bias in fp32.  Training is not
implemented: a forward with gradients enabled raises ValueError before any GPU work.
"""
import json
import os

import torch
import torch.nn as nn

from ... import ops
from ..hf_model import HFEncoder, ParamLayout, _normalise_config
from .colbert_model import _KINDS, encode_tokens
from .mlm_head import MaskedLMHeadMixin


class SPLADEEncoder(MaskedLMHeadMixin, nn.Module):
    def __init__(self, model_path: str = "roberta-base", dropout: float = 0.1, _config=None, _seed: int = 0):
        super().__init__()
        if _config is not None:
            raw, sd = dict(_config), None
        else:
            if not os.path.isdir(model_path):
                raise FileNotFoundError(f"model_path {model_path!r} is not a local directory "
                                        "(no network here: hub names cannot be resolved)")
            with open(os.path.join(model_path, "config.json")) as f:
                raw = json.load(f)
            self._check_config(raw)                   # fail before reading the weights
            _, sd = HFEncoder._read_pretrained(model_path)
        cfg = self._check_config(raw)
        if sd is None:
            body = HFEncoder(model_path="", dropout=dropout, _config=raw, _seed=_seed, _pooler=False)
        else:
            body = HFEncoder(model_path="", dropout=dropout, _config=raw, _state=sd, _pooler=False)
        self.config = cfg
        self.__dict__["_body"] = body   # not a submodule: its parameters are registered below, under the reference names
        self._build_head(body, cfg, sd)
        self.eval()

    @staticmethod
    def _check_config(raw):
        """Normalised config; ValueError for what the kernels cannot run, before any GPU work."""
        kind = raw.get("model_type", "bert")
        if kind not in _KINDS:
            raise ValueError(f"SPLADEEncoder supports BERT, RoBERTa and XLM-R encoders (model_type={kind!r})")
        cfg = _normalise_config(raw)
        ParamLayout(cfg)                  # head_dim 64, H / I multiples of 8, H <= 1024
        H = cfg["hidden_size"]
        ops.splade_pool_check(1, cfg["vocab_size"], H, H + 8, H + 8)
        return cfg

    @classmethod
    def from_config(cls, config, seed: int = 0):
        """Random init (HF scheme) from a config dict, without a checkpoint directory."""
        return cls(model_path="", dropout=0.0, _config=dict(config), _seed=seed)

    @property
    def dim(self):
        return self.config["vocab_size"]

    # ------------------------------------------------------------------ forward
    def _check_call(self, tokens):
        if torch.is_grad_enabled():
            raise ValueError("SPLADEEncoder runs forward only (training is not implemented): call it under "
                             "torch.no_grad()")
        S = tokens["input_ids"].shape[-1]
        if not 2 <= S <= ops.MAXSIM_MAX_S:
            raise ValueError(f"SPLADEEncoder needs 2 .. {ops.MAXSIM_MAX_S} tokens per sequence (got {S}): token 0 "
                             "is dropped")

    def forward(self, tokens):
        self._check_call(tokens)
        hidden, am, N, S = encode_tokens(self._body, tokens)
        keep = am != 0
        keep[:, 0] = False                                       # the reference pools tokens 1..
        rows = keep.view(-1).nonzero().squeeze(1)
        off = torch.zeros(N + 1, dtype=torch.int32, device=am.device)
        off[1:] = torch.cumsum(keep.sum(1), 0)
        H = self.config["hidden_size"]
        x = self.router_tokens(hidden[rows]) if rows.numel() else hidden.new_zeros(0, H + 8, dtype=torch.float16)
        return ops.splade_pool(x, self.router_operand(), off, H, self.router_bias().detach())
