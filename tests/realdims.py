"""Deterministic recipes for the parity cases at BASELINE.json's REAL model dimensions.

The weights are far too large to commit (BERT-base 0.44 GB, RoBERTa-large 1.4 GB), so both sides rebuild them from a
seed: `torch.manual_seed(0); BertModel(BertConfig())` (HF default init) for the query
encoder, the same + 0.01 * randn (`manual_seed(1)`) for the context encoder; RoBERTa-large from its published RobertaConfig.  `tests/golden/make_golden_realdims.py` runs the UNMODIFIED reference on them here and commits
embeddings / logits / loss / a sample of gradients + fp64 checksums of the weights; the GPU tests rebuild the weights on
the box, check the checksums (same torch + transformers => same RNG stream) and compare the CUDA path with the golden.
"""
import torch

BERT_BASE = dict(vocab_size=30522, hidden_size=768, num_hidden_layers=12, num_attention_heads=12,
                 intermediate_size=3072, max_position_embeddings=512, type_vocab_size=2, layer_norm_eps=1e-12,
                 pad_token_id=0)
ROBERTA_LARGE = dict(vocab_size=50265, hidden_size=1024, num_hidden_layers=24, num_attention_heads=16,
                     intermediate_size=4096, max_position_embeddings=514, type_vocab_size=1, layer_norm_eps=1e-5,
                     pad_token_id=1)

CASES = {
    # name: (kind, config, queries, hard negatives, seq len, temperature)
    # cfg 1 of BASELINE.json: 8 q + 16 ctx, S = 64, padded (variant B); T = 1 is the reference default
    "bert_base_cfg1": ("bert", BERT_BASE, 8, 1, 64, 1.0),
    # cfg 4's model at a batch the CPU reference finishes in seconds: 2 q + 4 ctx, S = 256, pad-derived positions
    "roberta_large_s256": ("roberta", ROBERTA_LARGE, 2, 1, 256, 1.0),
}


def hf_models(kind, cfg):
    """(query model, context model) as HF modules on the CPU, eval mode, dropout 0."""
    from transformers import BertConfig, BertModel, RobertaConfig, RobertaModel
    torch.manual_seed(0)
    if kind == "bert":
        q = BertModel(BertConfig(**cfg, hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0))
    else:
        q = RobertaModel(RobertaConfig(**cfg, hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0))
    import copy
    c = copy.deepcopy(q)
    g = torch.Generator().manual_seed(1)
    with torch.no_grad():
        for p in c.parameters():
            p.add_(0.01 * torch.randn(p.shape, generator=g))
    return q.eval(), c.eval()


def checksums(model):
    """Order-sensitive fp64 fingerprint of a model's parameters (detects any difference in the RNG stream)."""
    tot, wtot, n = 0.0, 0.0, 0
    for i, (k, p) in enumerate(sorted(model.state_dict().items())):
        if not p.dtype.is_floating_point:
            continue
        d = p.double()
        tot += float(d.sum())
        wtot += float((d.flatten()[::97] * (1 + (i % 7))).sum())
        n += p.numel()
    return torch.tensor([tot, wtot, float(n)], dtype=torch.float64)


def tokens(gen, n, S, pad_id, kind):
    """Benchmark inputs, variant B: lengths ~ U{S/4..S}, ids ~ U{1000..29999}, [CLS] first, [SEP] last real position."""
    lens = torch.randint(S // 4, S + 1, (n,), generator=gen)
    lens[0] = S
    ids = torch.randint(1000, 30000, (n, S), generator=gen)
    am = (torch.arange(S).unsqueeze(0) < lens.unsqueeze(1)).long()
    cls_id, sep_id = (101, 102) if kind == "bert" else (0, 2)
    ids[:, 0] = cls_id
    ids[torch.arange(n), lens - 1] = sep_id
    ids = ids * am + pad_id * (1 - am)
    out = {"input_ids": ids, "attention_mask": am}
    if kind == "bert":
        out["token_type_ids"] = torch.zeros_like(ids)
    return out


def batch(name, rank=0):
    kind, cfg, B, n, S, _ = CASES[name]
    gen = torch.Generator().manual_seed(1234 + rank)
    C = B * (1 + n)
    mask = torch.zeros(C, dtype=torch.bool)
    neg = torch.ones(C, dtype=torch.bool)
    neg[::1 + n] = False
    mask[neg] = torch.rand(int(neg.sum()), generator=gen) < 0.05
    if not mask.any():
        mask[1] = True                      # at least one dummy negative so the column predicate is exercised
    return {"query_ids": tokens(gen, B, S, cfg["pad_token_id"], kind),
            "contexts_ids": tokens(gen, C, S, cfg["pad_token_id"], kind),
            "pos_ctx_indices": torch.arange(B) * (1 + n), "ctx_mask": mask}


def sampled_grad_names(cfg):
    """The handful of gradient tensors whose reference values are committed (small ones + weight-matrix corners)."""
    L = cfg["num_hidden_layers"]
    names = ["embeddings.LayerNorm.weight", "embeddings.LayerNorm.bias", "embeddings.position_embeddings.weight"]
    for l in (0, L // 2, L - 1):
        p = f"encoder.layer.{l}."
        names += [p + "attention.self.query.bias", p + "attention.self.value.bias", p + "attention.output.dense.bias",
                  p + "attention.output.LayerNorm.weight", p + "intermediate.dense.bias", p + "output.dense.bias",
                  p + "output.LayerNorm.bias", p + "attention.self.query.weight", p + "intermediate.dense.weight",
                  p + "output.dense.weight"]
    return names


def sample(name, t):
    """Committed view of a gradient tensor: small tensors whole, matrices as their leading 48 x 48 corner."""
    if t.dim() == 2 and t.numel() > 70000:
        return t[:48, :48].contiguous()
    return t
