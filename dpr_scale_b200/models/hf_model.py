"""HFEncoder — drop-in for ``dpr_scale.models.hf_model.HFEncoder`` (/root/reference/dpr_scale/models/hf_model.py:12-41)
whose transformer arithmetic runs entirely in libdprb.so (hand-written sm_90a kernels).

Same constructor kwargs (``model_path, dropout, projection_dim``), same call signature
(``forward(tokens: Mapping) -> Tensor[N, d]``, fresh storage like the reference's ``.clone()``), same
``state_dict`` keys / shapes (``transformer.<hf names>``, ``project.0/1.*``) so Lightning checkpoints of the
reference load unchanged.

Storage: all transformer parameters are views into ONE flat fp32 "master" arena (HF layout, Q/K/V adjacent so
they form the fused [3H, H] weight); a bf16 shadow arena feeds the tensor-core GEMMs; gradients accumulate into a
flat fp32 arena whose views are exposed as ``param.grad``.  There is no CPU / eager fallback: ``forward`` on a
non-CUDA module raises.
"""
import ctypes
import json
import math
import os
from typing import Mapping, Optional

import torch
import torch.nn as nn

from .. import _lib, ops
from .._lib import EncoderBatch, EncoderWeights, check


# ----------------------------------------------------------------------------- layout
def _layer_entries(H, I):
    a = "attention."
    return [
        (a + "self.query.weight", (H, H)), (a + "self.key.weight", (H, H)), (a + "self.value.weight", (H, H)),
        (a + "self.query.bias", (H,)), (a + "self.key.bias", (H,)), (a + "self.value.bias", (H,)),
        (a + "output.dense.weight", (H, H)), (a + "output.dense.bias", (H,)),
        (a + "output.LayerNorm.weight", (H,)), (a + "output.LayerNorm.bias", (H,)),
        ("intermediate.dense.weight", (I, H)), ("intermediate.dense.bias", (I,)),
        ("output.dense.weight", (H, I)), ("output.dense.bias", (H,)),
        ("output.LayerNorm.weight", (H,)), ("output.LayerNorm.bias", (H,)),
    ]


class ParamLayout:
    """Element offsets of every HF parameter inside the flat arenas (mirrors dprb_encoder_weights)."""

    def __init__(self, cfg):
        H, I, L = cfg["hidden_size"], cfg["intermediate_size"], cfg["num_hidden_layers"]
        if H % 8 or I % 8 or H > 1024 or H // cfg["num_attention_heads"] != 64:
            raise ValueError(
                f"dprb kernels need head_dim 64, hidden/intermediate multiples of 8 and hidden <= 1024 "
                f"(got H={H}, I={I}, heads={cfg['num_attention_heads']})")
        self.cfg = cfg
        self.entries = []  # (name, shape, offset)
        off = 0

        def add(name, shape):
            nonlocal off
            n = int(math.prod(shape))
            assert n % 8 == 0, (name, shape)
            self.entries.append((name, tuple(shape), off))
            off += n

        e = "embeddings."
        add(e + "word_embeddings.weight", (cfg["vocab_size"], H))
        add(e + "position_embeddings.weight", (cfg["max_position_embeddings"], H))
        add(e + "token_type_embeddings.weight", (cfg["type_vocab_size"], H))
        add(e + "LayerNorm.weight", (H,))
        add(e + "LayerNorm.bias", (H,))
        self.off_layer0 = off
        for l in range(L):
            for name, shape in _layer_entries(H, I):
                add(f"encoder.layer.{l}.{name}", shape)
            if l == 0:
                self.layer_stride = off - self.off_layer0
        self.total = off
        self.by_name = {n: (s, o) for n, s, o in self.entries}

    def rel(self, name):
        return self.by_name["encoder.layer.0." + name][1] - self.off_layer0

    def fill_struct(self, w: EncoderWeights):
        c = self.cfg
        w.hidden, w.inter, w.layers = c["hidden_size"], c["intermediate_size"], c["num_hidden_layers"]
        w.heads, w.vocab = c["num_attention_heads"], c["vocab_size"]
        w.max_pos, w.type_vocab, w.ln_eps = c["max_position_embeddings"], c["type_vocab_size"], c["layer_norm_eps"]
        o = lambda n: self.by_name[n][1]
        w.off_word = o("embeddings.word_embeddings.weight")
        w.off_pos = o("embeddings.position_embeddings.weight")
        w.off_type = o("embeddings.token_type_embeddings.weight")
        w.off_emb_ln_g = o("embeddings.LayerNorm.weight")
        w.off_emb_ln_b = o("embeddings.LayerNorm.bias")
        w.off_layer0, w.layer_stride = self.off_layer0, self.layer_stride
        w.rel_wqkv = self.rel("attention.self.query.weight")
        w.rel_bqkv = self.rel("attention.self.query.bias")
        w.rel_wo, w.rel_bo = self.rel("attention.output.dense.weight"), self.rel("attention.output.dense.bias")
        w.rel_ln1_g, w.rel_ln1_b = self.rel("attention.output.LayerNorm.weight"), self.rel("attention.output.LayerNorm.bias")
        w.rel_w1, w.rel_b1 = self.rel("intermediate.dense.weight"), self.rel("intermediate.dense.bias")
        w.rel_w2, w.rel_b2 = self.rel("output.dense.weight"), self.rel("output.dense.bias")
        w.rel_ln2_g, w.rel_ln2_b = self.rel("output.LayerNorm.weight"), self.rel("output.LayerNorm.bias")


def _normalise_config(raw):
    cfg = dict(raw)
    cfg.setdefault("model_type", "bert")
    cfg.setdefault("type_vocab_size", 2)
    cfg.setdefault("layer_norm_eps", 1e-12)
    cfg.setdefault("pad_token_id", 1 if cfg["model_type"] in ("roberta", "xlm-roberta") else 0)
    cfg.setdefault("initializer_range", 0.02)
    act = cfg.get("hidden_act", "gelu")
    if act != "gelu":
        raise ValueError(f"dprb kernels implement erf-GELU only (hidden_act={act!r})")
    if cfg.get("position_embedding_type", "absolute") != "absolute":
        raise ValueError("only absolute position embeddings are supported")
    return cfg


def _set_nested(root: nn.Module, dotted: str, value):
    parts = dotted.split(".")
    m = root
    for p in parts[:-1]:
        if p not in m._modules:
            m.add_module(p, nn.Module())
        m = m._modules[p]
    if isinstance(value, nn.Parameter):
        m.register_parameter(parts[-1], value)
    else:
        m.register_buffer(parts[-1], value)


# ----------------------------------------------------------------------------- autograd glue
class _EncoderFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, master, enc, tokens, save):
        pooled, state = enc._run_forward(tokens, save)
        ctx.enc, ctx.state = enc, state
        return pooled

    @staticmethod
    def backward(ctx, dpooled):
        enc, state = ctx.enc, ctx.state
        ctx.state = None
        try:
            # shared_model=True: the same encoder back-propagates twice per step into one gradient arena; only the
            # LAST outstanding backward may hand finished slices to the trainer's all-reduce (trainer.py)
            enc._run_backward(state, dpooled.contiguous().float(), sync=enc._pending_bwd <= 1)
        finally:
            enc._pending_bwd = max(0, enc._pending_bwd - 1)
            state.release()
        return None, None, None, None


class _ChunkedEncoderFn(torch.autograd.Function):
    """Activation-memory bound for very large context batches (e.g. BASELINE config 4: 262 144 tokens x 24 layers of
    RoBERTa-large would need ~214 GB of saved activations): forward encodes `chunk` sequences at a time WITHOUT saving
    activations; backward re-runs each chunk with saving (same dropout seeds) and back-propagates its slice of the
    upstream gradient.  Mathematically identical to the unchunked path (the loss only sees the pooled embeddings)."""

    @staticmethod
    def forward(ctx, anchor, enc, tokens, chunk):
        n = tokens["input_ids"].shape[0]
        outs, seeds = [], []
        for lo in range(0, n, chunk):
            part = {k: v[lo:lo + chunk] for k, v in tokens.items() if v is not None}
            pooled, _ = enc._run_forward(part, False, train_dropout=True)
            seeds.append(enc.last_dropout[1])
            outs.append(pooled)
        ctx.enc, ctx.tokens, ctx.chunk, ctx.seeds = enc, tokens, chunk, seeds
        return torch.cat(outs, 0)

    @staticmethod
    def backward(ctx, dpooled):
        enc, tokens, chunk = ctx.enc, ctx.tokens, ctx.chunk
        dpooled = dpooled.contiguous().float()
        n = tokens["input_ids"].shape[0]
        starts = list(range(0, n, chunk))
        try:
            for i, lo in enumerate(starts):
                part = {k: v[lo:lo + chunk] for k, v in tokens.items() if v is not None}
                _, state = enc._run_forward(part, True, train_dropout=True, force_seed=ctx.seeds[i])
                # every chunk accumulates into the same arena: only the last chunk of the last outstanding backward
                # may release slices to the gradient all-reduce
                last = (i == len(starts) - 1) and enc._pending_bwd <= 1
                enc._run_backward(state, dpooled[lo:lo + chunk].contiguous(), sync=last)
                state.release()
        finally:
            enc._pending_bwd = max(0, enc._pending_bwd - 1)
        return None, None, None, None


class _ProjectFn(torch.autograd.Function):
    """``project = Sequential(Linear(H, p), LayerNorm(p))`` of hf_model.py:26-34 on the dprb kernels:
    pooled fp32 -> bf16 -> wgmma GEMM (+bias, bf16 out) -> dprb_ln_fwd whose fp32 row output IS the result;
    backward: dprb_ln_bwd (fused dgamma / dbeta / Linear-bias gradient) -> wgrad GEMM (fp32 split-K accumulate) and
    dgrad GEMM (fp32 store) back into the encoder's upstream gradient.  Same precision contract as the encoder body:
    16-bit GEMM operands, fp32 accumulation, fp32 LayerNorm statistics, fp32 parameters and gradients."""

    @staticmethod
    def forward(ctx, pooled, weight, bias, gamma, beta, eps):
        N, H = pooled.shape
        P = weight.shape[0]
        if P % 8 or P > 1024 or H % 8:
            raise ValueError(f"dprb projection head needs projection_dim % 8 == 0 and <= 1024 (got {P})")
        dev = pooled.device
        x16 = torch.empty(N, H, dtype=torch.bfloat16, device=dev)
        w16 = torch.empty(P, H, dtype=torch.bfloat16, device=dev)
        ops.cast_f32_bf16(pooled.contiguous(), x16)
        ops.cast_f32_bf16(weight.detach().contiguous(), w16)
        z = torch.empty(N, P, dtype=torch.bfloat16, device=dev)
        ops.gemm(x16, w16, z, N, P, H, H, H, P, False, False, ops.EPI_BIAS, bias.detach().contiguous())
        _, stats, out = ops.ln_fwd(z, gamma.detach().contiguous(), beta.detach().contiguous(), eps, cls_stride=1)
        ctx.save_for_backward(x16, w16, z, stats, gamma.detach())
        return out

    @staticmethod
    def backward(ctx, dout):
        x16, w16, z, stats, gamma = ctx.saved_tensors
        N, H = x16.shape
        P = w16.shape[0]
        dev = x16.device
        dgamma, dbeta, dbias = (torch.zeros(P, dtype=torch.float32, device=dev) for _ in range(3))
        dz = ops.ln_bwd(None, z, stats, gamma.contiguous(), dgamma, dbeta, dbias, dy_cls=dout.contiguous().float(),
                        cls_stride=1)
        dw = torch.zeros(P, H, dtype=torch.float32, device=dev)
        ops.gemm(dz, x16, dw, P, H, N, P, H, H, True, True, ops.EPI_F32_ATOMIC_ADD, None, splits=0)
        dx = torch.empty(N, H, dtype=torch.float32, device=dev)
        ops.gemm(dz, w16, dx, N, H, P, P, H, H, False, True, ops.EPI_F32_STORE, None)
        return dx, dw, dbias, dgamma, dbeta, None


class _FwdState:
    """What one forward hands to its backward: the C structs, the token tensors they point into, and a LEASE on the
    activation workspace.  The workspace goes back to the encoder's pool when the state is released (end of backward)
    or garbage-collected (a forward whose graph is dropped) - never while a backward may still read it, so two live
    forwards of one encoder (shared_model=True: query + context pass of equal shape) cannot alias."""

    __slots__ = ("w", "b", "keep", "ws", "_pool")

    def __init__(self, w, b, keep, ws, pool):
        self.w, self.b, self.keep, self.ws, self._pool = w, b, keep, ws, pool

    def release(self):
        ws, pool = self.ws, self._pool
        self.ws = self._pool = None
        if ws is not None and pool is not None:
            pool.give_back(ws)

    def __del__(self):
        try:
            self.release()
        except Exception:
            pass


class _WorkspacePool:
    """At most ONE idle buffer is kept (they are tens of GB); a lease takes it when it is large enough."""

    def __init__(self):
        self.idle = None
        self.leased = 0

    def lease(self, nbytes, device):
        buf = self.idle
        if buf is not None and buf.numel() >= nbytes and buf.device == device:
            self.idle = None
        else:
            self.idle = None          # too small / wrong device: let the allocator have it back first
            buf = torch.empty(nbytes, dtype=torch.uint8, device=device)
        self.leased += 1
        return buf

    def give_back(self, buf):
        self.leased -= 1
        if self.idle is None or self.idle.numel() < buf.numel():
            self.idle = buf


class _Transformer(nn.Module):
    """Container that owns the arenas and mirrors the HF module tree (parameter names only)."""

    def __init__(self, cfg, master: torch.Tensor, pooler: bool = True):
        super().__init__()
        self.cfg = cfg
        self.layout = ParamLayout(cfg)
        assert master.numel() == self.layout.total
        self._bind(master)
        H = cfg["hidden_size"]
        # HF's pooler is part of the reference state_dict but never used (hf_model.py:39) and gets no grad.  A BERT
        # cross-encoder uses it as the first layer of its classification head; RoBERTa's has none (pooler=False).
        if pooler:
            self.add_module("pooler", nn.Module())
            self.pooler.add_module("dense", nn.Linear(H, H))
        # Checkpoints written with the reference's pinned transformers==3.4.0 carry the persistent buffer
        # `embeddings.position_ids` (later releases made it non-persistent); it holds arange(max_pos) and is not a
        # weight, so it is dropped on load instead of failing a strict load_state_dict.
        self._register_load_state_dict_pre_hook(self._drop_position_ids)

    @staticmethod
    def _drop_position_ids(state_dict, prefix, *unused):
        for k in (prefix + "embeddings.position_ids", prefix + "embeddings.token_type_ids"):
            state_dict.pop(k, None)

    def _bind(self, master):
        """(Re)create every parameter as a view into `master`."""
        self.__dict__["_master"] = master
        self.__dict__["_shadow"] = None
        self.__dict__["_grads"] = None
        self.__dict__["_shadow_version"] = -1
        for name, shape, off in self.layout.entries:
            view = master[off:off + math.prod(shape)].view(shape)
            _set_nested(self, name, nn.Parameter(view, requires_grad=True))

    def _apply(self, fn, recurse=True):
        master = fn(self._master)
        if master.dtype != torch.float32:
            raise TypeError("dprb encoder master weights must stay fp32 (bf16 shadows are managed internally)")
        if "pooler" in self._modules:
            self.pooler._apply(fn)
        self._bind(master)
        return self

    def arena_params(self):
        for name, shape, off in self.layout.entries:
            m = self
            for p in name.split("."):
                m = getattr(m, p)
            yield name, m, off


class HFEncoder(nn.Module):
    def __init__(self, model_path: str = "roberta-base", dropout: float = 0.1,
                 projection_dim: Optional[int] = None, _config=None, _seed: Optional[int] = None, _state=None,
                 _pooler: bool = True):
        super().__init__()
        if _config is not None and _state is not None:     # config + HF state dict already read by the caller
            cfg, sd = _normalise_config(_config), _state
            master = torch.zeros(ParamLayout(cfg).total, dtype=torch.float32)
        elif _config is not None:
            cfg = _normalise_config(_config)
            master = self._random_init(cfg, _seed if _seed is not None else 0)
            sd = None
        else:
            cfg, sd = self._read_pretrained(model_path)
            master = torch.zeros(ParamLayout(cfg).total, dtype=torch.float32)
        self.config = cfg
        self.dropout = float(dropout)
        self.transformer = _Transformer(cfg, master, pooler=_pooler)
        if sd is not None:
            self._load_hf_state(sd)
        self.project = nn.Identity()
        if projection_dim == -1:
            projection_dim = cfg["hidden_size"]
        if projection_dim:
            linear = nn.Linear(cfg["hidden_size"], projection_dim)
            linear.weight.data.normal_(mean=0.0, std=0.02)
            self.project = nn.Sequential(linear, nn.LayerNorm(projection_dim))
        self._ws_cache = {}                  # forward-only workspaces (consumed before forward returns)
        self._ws_pool = _WorkspacePool()     # save-for-backward workspaces, leased per live forward
        self._pending_bwd = 0                # forwards of this step whose backward has not run yet
        self._warned_dropout = False
        self.launches = 0
        # multi-GPU hook (set by the trainer): backward runs in `bwd_chunk_layers`-layer chunks and calls
        # grad_sync(lo_elem, hi_elem) after each chunk so the gradient all-reduce of the finished slice of the
        # flat arena overlaps with the rest of backward.
        self.grad_sync = None
        self.bwd_chunk_layers = 0
        self._drop_base = (torch.initial_seed() * 0x9E3779B97F4A7C15 + id(self)) & 0xFFFFFFFFFFFFFFFF
        self._drop_calls = 0
        # sequences per activation chunk (0 = keep all activations of the batch; see _ChunkedEncoderFn)
        self.activation_chunk = int(os.environ.get("DPRB_ACTIVATION_CHUNK", "0"))
        # lean activations (dprb_encoder_batch.save_for_backward = 2): keep the FFN pre-activation instead of
        # gelu + gelu' and no attention output; backward rebuilds them (one elementwise pass + one attention forward per
        # layer).  22 KB instead of 32 KB per token and layer at RoBERTa-large: BASELINE config 4 fits without recompute.
        self.lean_activations = bool(int(os.environ.get("DPRB_LEAN_ACTIVATIONS", "0")))

    # ------------------------------------------------------------------ construction helpers
    @classmethod
    def from_config(cls, config: Mapping, dropout: float = 0.1, projection_dim: Optional[int] = None, seed: int = 0):
        """Random-init (HF scheme: N(0, initializer_range), LN = 1/0, biases 0) without a checkpoint directory."""
        return cls(model_path="", dropout=dropout, projection_dim=projection_dim, _config=dict(config), _seed=seed)

    @staticmethod
    def _random_init(cfg, seed):
        layout = ParamLayout(cfg)
        g = torch.Generator().manual_seed(seed)
        master = torch.empty(layout.total, dtype=torch.float32)
        for name, shape, off in layout.entries:
            n = math.prod(shape)
            v = master[off:off + n]
            if "LayerNorm.weight" in name:
                v.fill_(1.0)
            elif name.endswith("bias"):
                v.zero_()
            else:
                v.normal_(0.0, cfg["initializer_range"], generator=g)
        o = layout.by_name["embeddings.word_embeddings.weight"][1]
        H = cfg["hidden_size"]
        master[o + cfg["pad_token_id"] * H: o + (cfg["pad_token_id"] + 1) * H].zero_()
        return master

    @staticmethod
    def _read_pretrained(model_path):
        path = model_path
        if not os.path.isdir(path):
            raise FileNotFoundError(
                f"model_path {model_path!r} is not a local directory (no network here: hub names cannot be resolved)")
        with open(os.path.join(path, "config.json")) as f:
            cfg = _normalise_config(json.load(f))
        st = os.path.join(path, "model.safetensors")
        if os.path.exists(st):
            from safetensors.torch import load_file
            sd = load_file(st)
        else:
            sd = torch.load(os.path.join(path, "pytorch_model.bin"), map_location="cpu")
        return cfg, sd

    def _load_hf_state(self, sd):
        own = self.transformer.state_dict()
        fixed = {}
        for k, v in sd.items():
            for pre in ("bert.", "roberta.", "transformer."):
                if k.startswith(pre):
                    k = k[len(pre):]
            k = k.replace("LayerNorm.gamma", "LayerNorm.weight").replace("LayerNorm.beta", "LayerNorm.bias")
            if k in own:
                fixed[k] = v
        missing = [k for k in own if k not in fixed and not k.startswith("pooler.")]
        if missing:
            raise KeyError(f"checkpoint is missing encoder weights: {missing[:5]} ...")
        self.transformer.load_state_dict(fixed, strict=False)

    # ------------------------------------------------------------------ arenas
    @property
    def master(self):
        return self.transformer._master

    def _ensure_device_state(self, need_grads):
        t = self.transformer
        m = t._master
        if not m.is_cuda:
            raise _lib.DprbError("HFEncoder (dprb) runs on CUDA only — move the module to an H100 (`.cuda()`); "
                                 "there is no CPU fallback")
        if t._shadow is None or t._shadow.device != m.device:
            t.__dict__["_shadow"] = torch.empty(m.numel(), dtype=torch.bfloat16, device=m.device)
            t.__dict__["_shadow_version"] = -1
        if t._shadow_version != m._version:
            ops.cast_f32_bf16(m, t._shadow)
            self.launches += 1
            t.__dict__["_shadow_version"] = m._version
        if need_grads and (t._grads is None or t._grads.device != m.device):
            t.__dict__["_grads"] = torch.zeros(m.numel(), dtype=torch.float32, device=m.device)
            for name, p, off in t.arena_params():
                p.grad = t._grads[off:off + p.numel()].view(p.shape)

    def mark_shadow_fresh(self):
        """Called by the fused optimizer, which rewrites master and shadow in the same kernel."""
        self.transformer.__dict__["_shadow_version"] = self.transformer._master._version

    @property
    def grads(self):
        self._ensure_device_state(True)
        return self.transformer._grads

    @property
    def shadow(self):
        self._ensure_device_state(False)
        return self.transformer._shadow

    def zero_grad(self, set_to_none: bool = False):
        # gradients live in the flat arena (kernels accumulate with atomics): always zero in place
        if self.transformer._grads is not None:
            self.transformer._grads.zero_()
        self._pending_bwd = 0   # a forward that was never back-propagated must not block next step's gradient sync
        for p in self.project.parameters():
            p.grad = None

    def _weights_struct(self, with_grads):
        w = EncoderWeights()
        self.transformer.layout.fill_struct(w)
        t = self.transformer
        w.master = t._master.data_ptr()
        w.shadow = t._shadow.data_ptr()
        w.grads = t._grads.data_ptr() if (with_grads and t._grads is not None) else None
        return w

    def _save_mode(self, save):
        return 0 if not save else (2 if self.lean_activations else 1)

    def _workspace(self, nseq, S, save):
        w = self._weights_struct(False)
        nbytes = _lib.load().dprb_encoder_workspace_bytes(ctypes.byref(w), nseq, S, self._save_mode(save))
        if nbytes < 0:
            check(1, "dprb_encoder_workspace_bytes")
        if save:
            # saved activations live here until backward: one lease per live forward (see _FwdState)
            return self._ws_pool.lease(nbytes + 256, self.master.device)
        # forward-only: the buffer is dead when forward returns (the pooled output is a separate tensor), so one
        # cached buffer per stream is enough; shapes vary batch to batch (pad-to-longest) and the buffers are large
        key = torch.cuda.current_stream().cuda_stream
        ws = self._ws_cache.get(key)
        if ws is None or ws.numel() < nbytes + 256 or ws.device != self.master.device:
            self._ws_cache.pop(key, None)
            ws = torch.empty(nbytes + 256, dtype=torch.uint8, device=self.master.device)
            self._ws_cache[key] = ws
        return ws

    # ------------------------------------------------------------------ forward / backward
    def _prep_tokens(self, tokens):
        ids = tokens["input_ids"]
        if ids.dim() != 2:
            raise ValueError("input_ids must be [N, S]")
        dev = self.master.device
        ids = ids.to(dev, torch.int64).contiguous()
        N, S = ids.shape
        # position ids must index the position table (HF raises an IndexError there); RoBERTa's are pad-derived and
        # reach S + pad_token_id.  The attention kernels stop at 512 tokens.
        max_pos = self.config["max_position_embeddings"]
        roberta = self.config["model_type"] in ("roberta", "xlm-roberta")
        limit = max_pos - self.config["pad_token_id"] - 1 if roberta else max_pos
        if S > limit:
            raise ValueError(f"sequence length {S} needs position ids beyond max_position_embeddings={max_pos} "
                             f"(longest supported: {limit})")
        if S > 512:
            raise ValueError(f"sequence length {S} unsupported: the dprb kernels take at most 512 tokens")
        tt = tokens.get("token_type_ids") if hasattr(tokens, "get") else None
        tt = torch.zeros_like(ids) if tt is None else tt.to(dev, torch.int64).contiguous()
        am = tokens.get("attention_mask") if hasattr(tokens, "get") else None
        am32 = None if am is None else am.to(dev, torch.int32).contiguous()
        if self.config["model_type"] in ("roberta", "xlm-roberta"):
            pad = self.config["pad_token_id"]
            m = (ids != pad).to(torch.int64)
            pos = torch.cumsum(m, dim=1) * m + pad  # modeling_roberta.py:146-159
        else:
            pos = torch.arange(S, device=dev, dtype=torch.int64).unsqueeze(0).expand(N, S)
        return ids, tt, pos.contiguous(), am32, N, S

    def _run_forward(self, tokens, save, train_dropout=None, force_seed=None):
        ids, tt, pos, am, N, S = self._prep_tokens(tokens)
        self._ensure_device_state(save)
        ws = self._workspace(N, S, save)
        base = (ws.data_ptr() + 255) & ~255
        b = EncoderBatch()
        b.nseq, b.S = N, S
        b.ids, b.type_ids, b.pos_ids = ids.data_ptr(), tt.data_ptr(), pos.data_ptr()
        b.attn_mask = am.data_ptr() if am is not None else None
        b.workspace, b.workspace_bytes = base, ws.numel() - (base - ws.data_ptr())
        b.save_for_backward = self._save_mode(save)
        # HF applies dropout only in train mode; the seed changes every forward and is replayed by backward
        use_drop = (self.training and save) if train_dropout is None else (self.training and train_dropout)
        b.dropout_p = self.dropout if use_drop else 0.0
        self._drop_calls += 1
        b.dropout_seed = force_seed if force_seed is not None else (
            (self._drop_base + self._drop_calls * 0x2545F4914F6CDD1D) & 0xFFFFFFFFFFFFFFFF)
        self.last_dropout = (float(b.dropout_p), int(b.dropout_seed))  # exposed for tests (mask reconstruction)
        w = self._weights_struct(save)
        pooled = torch.empty(N, self.config["hidden_size"], dtype=torch.float32, device=ids.device)
        stream = torch.cuda.current_stream().cuda_stream
        check(_lib.load().dprb_encoder_fwd(ctypes.byref(w), ctypes.byref(b), pooled.data_ptr(), stream),
              "dprb_encoder_fwd")
        L = self.config["num_hidden_layers"]
        self.launches += 1 + 7 * L
        return pooled, _FwdState(w, b, (ids, tt, pos, am), ws if save else None, self._ws_pool if save else None)

    def _run_backward(self, state, dpooled, sync=True):
        w, b = state.w, state.b
        L = self.config["num_hidden_layers"]
        stream = torch.cuda.current_stream().cuda_stream
        lay = self.transformer.layout
        sync = sync and self.grad_sync is not None
        if sync and self.bwd_chunk_layers > 0:
            # buckets of `step` layers from the top; the last bucket is layer 0 alone, because it also carries the
            # embedding tables (22 % of BERT-base) and is the only one whose all-reduce cannot hide behind backward
            step = self.bwd_chunk_layers
            bounds = [(max(1, hi - step), hi) for hi in range(L, 1, -step)] + [(0, 1)]
            bounds = [b for b in bounds if b[0] < b[1]]
        else:
            bounds = [(0, L)]
        for lo, hi in bounds:
            check(_lib.load().dprb_encoder_bwd(ctypes.byref(w), ctypes.byref(b), dpooled.data_ptr(), lo, hi, stream),
                  "dprb_encoder_bwd")
            if sync:
                e_lo = 0 if lo == 0 else lay.off_layer0 + lo * lay.layer_stride  # lo == 0 also finishes the embeddings
                self.grad_sync(self, e_lo, lay.off_layer0 + hi * lay.layer_stride)

    def forward(self, tokens):
        save = torch.is_grad_enabled()
        if save:
            # any arena parameter works as the autograd anchor; gradients are written by the kernels
            # straight into the flat grads arena (exposed as param.grad views), so backward returns None.
            anchor = self.transformer.embeddings.LayerNorm.weight
            n = tokens["input_ids"].shape[0]
            if self.activation_chunk and n > self.activation_chunk:
                tk = {k: tokens[k] for k in ("input_ids", "token_type_ids", "attention_mask") if k in tokens}
                self._pending_bwd += 1
                rep = _ChunkedEncoderFn.apply(anchor, self, tk, self.activation_chunk)
            else:
                self._pending_bwd += 1
                rep = _EncoderFn.apply(anchor, self, tokens, True)
        else:
            rep, _ = self._run_forward(tokens, False)
        if not isinstance(self.project, nn.Identity):
            lin, ln = self.project[0], self.project[1]
            rep = _ProjectFn.apply(rep, lin.weight, lin.bias, ln.weight, ln.bias, ln.eps)
        return rep  # already fresh storage (reference: sentence_rep.clone())
