"""The masked-LM head shared by CITADELEncoder (its router) and SPLADEEncoder (its vocabulary pooling).

State-dict layout, as HF's ``BertForMaskedLM`` / ``RobertaForMaskedLM`` under ``transformer.``:
``transformer.bert.*`` (no pooler) and ``transformer.cls.predictions.{bias, transform.dense.*, transform.LayerNorm.*,
decoder.weight, decoder.bias}`` for BERT, ``transformer.roberta.*`` and ``transformer.lm_head.{bias, dense.*,
layer_norm.*, decoder.weight, decoder.bias}`` for RoBERTa / XLM-R.  As in HF, the decoder is tied: its weight IS the
word-embedding table and its bias IS the head's bias, so both appear under two names and load through the body / head
keys.

What runs: the head's dense layer + GELU is the library's GEMM with the bias-GELU epilogue and its LayerNorm is
``dprb_ln_fwd`` (fp16 output), giving ``head_tokens`` [T, H + 8]; the decoder operand ``head_operand`` [V, H + 8] (built
once per weight version and cached) holds the word embeddings with the fp16 decoder bias in column H, so with the 1 the
tokens carry there an fp32-accumulated inner product over H + 1 columns is the logit.  Both operands are fp16 (11
significant bits against bf16's 8).
"""
import torch
import torch.nn as nn

from ... import ops

HEAD_DTYPE = torch.float16


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


class MaskedLMHeadMixin:
    """For an nn.Module with an HFEncoder body (``_body``, built with ``_pooler=False``): ``_build_head`` registers the
    body and the head under the HF masked-LM names; the other methods run the head."""

    def _build_head(self, body, cfg, sd):
        """Registers ``transformer.{bert|roberta}`` and the head (HF init: dense N(0, initializer_range), biases 0,
        LayerNorm 1 / 0), then copies the head of the HF state dict ``sd`` where it has one."""
        H, V = cfg["hidden_size"], cfg["vocab_size"]
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

    def word_embeddings(self):
        return self._body.transformer.embeddings.word_embeddings.weight

    def router_bias(self):
        return self._head.bias

    def _head_layers(self):
        h = self._head
        return (h.transform.dense, h.transform.LayerNorm) if self.bert_head else (h.dense, h.layer_norm)

    def router_operand(self):
        """[V, H + 8] HEAD_DTYPE: the decoder rows (the word embeddings) with the decoder bias in column H and zeros
        after it; rebuilt only when the weights change."""
        word, bias = self.word_embeddings(), self.router_bias()
        key = (word.data_ptr(), word._version, bias.data_ptr(), bias._version)
        cache = self._router_cache
        if cache is not None and cache[0] == key:
            return cache[1]
        V, H = word.shape
        op = torch.zeros(V, H + 8, dtype=HEAD_DTYPE, device=word.device)
        op[:, :H] = word.detach()
        op[:, H] = bias.detach()
        self.__dict__["_router_cache"] = (key, op)
        return op

    def router_tokens(self, hidden):
        """[T, H + 8] HEAD_DTYPE: the head's transform (dense + GELU on the GEMM epilogue, LayerNorm) of hidden bf16
        [T, H], with 1 in column H (it picks up the bias column of the operand) and zeros after it."""
        dense, norm = self._head_layers()
        T, H = hidden.shape
        w16 = torch.empty(H, H, dtype=torch.bfloat16, device=hidden.device)
        ops.cast_f32_bf16(dense.weight.detach().contiguous(), w16)
        act = ops.linear_fwd(hidden, w16, dense.bias.detach().contiguous(), ops.EPI_BIAS_GELU)
        y16 = torch.empty(T, H, dtype=torch.float16, device=hidden.device)
        ops.ln_fwd(act, norm.weight.detach().contiguous(), norm.bias.detach().contiguous(), norm.eps, y_res=y16)
        x = torch.zeros(T, H + 8, dtype=HEAD_DTYPE, device=hidden.device)
        x[:, :H] = y16
        x[:, H] = 1.0
        return x
