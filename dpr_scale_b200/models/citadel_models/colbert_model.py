"""ColBERTEncoder — drop-in for ``dpr_scale.models.citadel_models.colbert_model.ColBERTEncoder``
(/root/reference/dpr_scale/models/citadel_models/colbert_model.py:12-44): a BERT or RoBERTa late-interaction encoder,
forward only.

Same constructor (``model_path, dropout, projection_dim``), same call (``forward(tokens) -> {"expert_repr": fp32
[N, S-1, P]}``: the last layer without token 0, projected, multiplied by ``attention_mask[:, 1:]`` so padded tokens are
exact zero vectors), same ``state_dict`` keys and shapes as the reference's ``transformer = AutoModel(...)`` (pooler
included) and ``project = Sequential(Linear(H, P))`` - no LayerNorm, unlike HFEncoder's head; ``projection_dim=None``
is the identity (P = H) and ``-1`` a Linear(H, H).  Reference checkpoints load strictly.

What runs: the encoder body is HFEncoder's arena and forward-only workspace; ``dprb_encoder_fwd_tokens`` writes every
token of the last layer in bf16 and the projection is the library's GEMM with the bias epilogue (bf16 out).
``token_reps`` returns those projected tokens with their mask, unmasked, for ``dprb_maxsim_fwd`` (which reads the masks
itself); ``forward`` builds the reference's masked fp32 tensor from them.  Training is not implemented: a forward with
gradients enabled raises ValueError before any GPU work.
"""
import json
import os
from typing import Optional

import torch
import torch.nn as nn

from ... import ops
from ..._lib import EncoderBatch
from ..hf_model import HFEncoder, ParamLayout, _normalise_config

_KINDS = ("bert", "roberta", "xlm-roberta")


def encode_tokens(body: HFEncoder, tokens):
    """(hidden bf16 [N*S, H], mask int32 [N, S], N, S): every token of the last layer of ``body``
    (dprb_encoder_fwd_tokens, eval mode)."""
    ids, tt, pos, am, N, S = body._prep_tokens(tokens)
    body._ensure_device_state(False)
    ws = body._workspace(N, S, False)
    base = (ws.data_ptr() + 255) & ~255
    b = EncoderBatch()
    b.nseq, b.S = N, S
    b.ids, b.type_ids, b.pos_ids = ids.data_ptr(), tt.data_ptr(), pos.data_ptr()
    b.attn_mask = am.data_ptr() if am is not None else None
    b.workspace, b.workspace_bytes = base, ws.numel() - (base - ws.data_ptr())
    b.save_for_backward, b.dropout_p, b.dropout_seed = 0, 0.0, 0      # eval: dropout is the identity
    H = body.config["hidden_size"]
    hidden = torch.empty(N * S, H, dtype=torch.bfloat16, device=ids.device)
    ops.encoder_fwd_tokens(body._weights_struct(False), b, hidden)
    body.launches += 1 + 7 * body.config["num_hidden_layers"]
    if am is None:
        am = torch.ones(N, S, dtype=torch.int32, device=ids.device)
    return hidden, am, N, S


def linear_bf16(lin: nn.Linear, x):
    """bf16 [T, out] = x @ lin.weight^T + lin.bias: x bf16 [T, in] contiguous, on the library's GEMM (bias epilogue)."""
    T, K = x.shape
    N = lin.out_features
    w16 = torch.empty(N, K, dtype=torch.bfloat16, device=x.device)
    ops.cast_f32_bf16(lin.weight.detach().contiguous(), w16)
    y = torch.empty(T, N, dtype=torch.bfloat16, device=x.device)
    ops.gemm(x, w16, y, T, N, K, K, K, N, False, False, ops.EPI_BIAS, lin.bias.detach().contiguous())
    return y


class ColBERTEncoder(nn.Module):
    def __init__(self, model_path: str = "roberta-base", dropout: float = 0.1, projection_dim: Optional[int] = None,
                 _config=None, _seed: int = 0):
        super().__init__()
        if _config is not None:
            raw, sd = dict(_config), None
        else:
            if not os.path.isdir(model_path):
                raise FileNotFoundError(f"model_path {model_path!r} is not a local directory "
                                        "(no network here: hub names cannot be resolved)")
            with open(os.path.join(model_path, "config.json")) as f:
                raw = json.load(f)
            self._check_config(raw, projection_dim)       # fail before reading the weights
            _, sd = HFEncoder._read_pretrained(model_path)
        cfg = self._check_config(raw, projection_dim)
        H = cfg["hidden_size"]
        if sd is None:
            body = HFEncoder(model_path="", dropout=dropout, _config=raw, _seed=_seed)
        else:
            body = HFEncoder(model_path="", dropout=dropout, _config=raw, _state=sd)
        self.config = cfg
        self.__dict__["_body"] = body  # not a submodule: its parameters are registered below, under the reference names
        self.transformer = body.transformer
        self.project = nn.Identity()
        if projection_dim == -1:
            projection_dim = H
        if projection_dim:
            linear = nn.Linear(H, projection_dim)
            linear.weight.data.normal_(mean=0.0, std=0.02)
            self.project = nn.Sequential(linear)
        self.eval()

    @staticmethod
    def _check_config(raw, projection_dim):
        """Normalised config; ValueError for what the kernels cannot run, before any GPU work."""
        kind = raw.get("model_type", "bert")
        if kind not in _KINDS:
            raise ValueError(f"ColBERTEncoder supports BERT, RoBERTa and XLM-R encoders (model_type={kind!r})")
        cfg = _normalise_config(raw)
        ParamLayout(cfg)                  # head_dim 64, H / I multiples of 8, H <= 1024
        P = cfg["hidden_size"] if projection_dim in (None, 0, -1) else int(projection_dim)
        ops.maxsim_check(2, 2, P)
        return cfg

    @classmethod
    def from_config(cls, config, projection_dim: Optional[int] = None, seed: int = 0):
        """Random init (HF scheme) from a config dict, without a checkpoint directory."""
        return cls(model_path="", dropout=0.0, projection_dim=projection_dim, _config=dict(config), _seed=seed)

    @property
    def dim(self):
        return self.project[0].out_features if isinstance(self.project, nn.Sequential) else self.config["hidden_size"]

    # ------------------------------------------------------------------ forward
    def _check_call(self, tokens):
        if torch.is_grad_enabled():
            raise ValueError(f"{type(self).__name__} runs forward only (training is not implemented): call it under "
                             "torch.no_grad()")
        S = tokens["input_ids"].shape[-1]
        if not 2 <= S <= ops.MAXSIM_MAX_S:
            raise ValueError(f"{type(self).__name__} needs 2 .. {ops.MAXSIM_MAX_S} tokens per sequence (got {S}): "
                             "token 0 is dropped")

    def token_reps(self, tokens):
        """(reps bf16 [N, S, P], mask int32 [N, S]): projected last-layer tokens, token 0 included and padded tokens not
        zeroed (their mask is 0)."""
        hidden, am, N, S = self._hidden(tokens)
        H = self.config["hidden_size"]
        if isinstance(self.project, nn.Identity):
            return hidden.view(N, S, H), am
        reps = linear_bf16(self.project[0], hidden)
        return reps.view(N, S, -1), am

    def _hidden(self, tokens):
        """(hidden bf16 [N*S, H], mask int32 [N, S], N, S): the last layer of every token."""
        self._check_call(tokens)
        return encode_tokens(self._body, tokens)

    def forward(self, tokens, **kwargs):
        reps, am = self.token_reps(tokens)
        keep = am[:, 1:].unsqueeze(-1) != 0
        expert = torch.where(keep, reps[:, 1:, :].float(), torch.zeros((), device=reps.device))
        return {"expert_repr": expert}
