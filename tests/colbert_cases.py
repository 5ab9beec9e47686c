"""Deterministic recipes shared by the ColBERT goldens (tests/golden/make_golden_colbert.py) and their tests: tiny BERT /
RoBERTa ColBERT encoders (with a 128-wide projection or none), single-sequence tokens, the rerank task's checkpoint and
the BERT-base-dims encoder.  No weights are committed: every state dict is rebuilt from its seed here (same torch +
transformers => same RNG stream), and the goldens hold fp64 checksums that prove it is the one the reference ran.
The fixture run, tokenizer and datamodule settings are those of tests/rerank_cases.py."""
import torch

from tests import rerank_cases
from tests.realdims import BERT_BASE, checksums  # noqa: F401

# name: (encoder kind, projection_dim, seed)
TINY = {"bert_p128": ("bert", 128, 31), "bert_none": ("bert", None, 32),
        "roberta_p128": ("roberta", 128, 33), "roberta_none": ("roberta", None, 34)}
TASK_KINDS = ("bert_p128", "roberta_p128")       # the rerank task's encoders (shared_model: false)
POOLS = ("sum", "max")
BASE_PAIRS, BASE_SQ, BASE_SD, BASE_P = 16, 32, 256, 128


def encoder_config(kind):
    """The tiny encoder configs of tests/rerank_cases.py without the classification labels."""
    cfg = rerank_cases.tiny_config(kind)
    cfg.pop("num_labels")
    return cfg


def state_dict(cfg, proj, seed):
    """A ColBERTEncoder state dict: ``transformer.*`` of a seeded HF BertModel / RobertaModel (HF init, then non-trivial
    biases and LayerNorm affines) + ``project.0.*`` when proj is set (weight std 0.05, bias std 0.02)."""
    from transformers import BertConfig, BertModel, RobertaConfig, RobertaModel
    torch.manual_seed(seed)
    if cfg["model_type"] == "bert":
        model = BertModel(BertConfig(**cfg))
    else:
        model = RobertaModel(RobertaConfig(**cfg))
    g = torch.Generator().manual_seed(seed + 100)
    with torch.no_grad():
        for name, p in model.named_parameters():
            if name.endswith("bias"):
                p.copy_(0.02 * torch.randn(p.shape, generator=g))
            elif "LayerNorm.weight" in name:
                p.copy_(1.0 + 0.02 * torch.randn(p.shape, generator=g))
    sd = {"transformer." + k: v.detach().clone() for k, v in model.state_dict().items()
          if not k.endswith(("position_ids", "token_type_ids"))}
    if proj:
        H = cfg["hidden_size"]
        sd["project.0.weight"] = 0.05 * torch.randn(proj, H, generator=g)
        sd["project.0.bias"] = 0.02 * torch.randn(proj, generator=g)
    return sd


def tiny_state_dict(name, seed_offset=0):
    kind, proj, seed = TINY[name]
    return state_dict(encoder_config(kind), proj, seed + seed_offset)


def task_state_dict(name):
    """The rerank task's checkpoint state dict: two different encoders of kind `name` (query: its seed, context: the
    seed + 1000)."""
    sd = {"query_encoder." + k: v for k, v in tiny_state_dict(name).items()}
    sd.update({"context_encoder." + k: v for k, v in tiny_state_dict(name, 1000).items()})
    return sd


def model_dir(path, name):
    """A checkpoint directory the reference's and this repo's ColBERTEncoder both load (plus the fixture tokenizer)."""
    from transformers import BertConfig, BertModel, RobertaConfig, RobertaModel
    kind, _, _ = TINY[name]
    cfg = encoder_config(kind)
    model = BertModel(BertConfig(**cfg)) if kind == "bert" else RobertaModel(RobertaConfig(**cfg))
    model.load_state_dict({k[len("transformer."):]: v for k, v in tiny_state_dict(name).items()
                           if k.startswith("transformer.")}, strict=False)
    model.save_pretrained(path)
    return rerank_cases.tokenizer_dir(path)


def seq_tokens(gen, n, S, vocab, pad_id, lo=5, cls_id=2, sep_id=3, min_len=None):
    """[CLS] text [SEP] pad..., token types 0; row 0 is full length, the others ~ U{min_len (default S/3)..S}."""
    lens = torch.randint(max(3, S // 3) if min_len is None else min_len, S + 1, (n,), generator=gen)
    lens[0] = S
    ids = torch.randint(lo, vocab, (n, S), generator=gen)
    for i in range(n):
        ids[i, 0], ids[i, int(lens[i]) - 1] = cls_id, sep_id
    am = (torch.arange(S).unsqueeze(0) < lens.unsqueeze(1)).long()
    ids = ids * am + pad_id * (1 - am)
    return {"input_ids": ids, "token_type_ids": torch.zeros_like(ids), "attention_mask": am}


def bert_base_state_dict():
    """(state dict, config): BERT-base dims, the recipe of state_dict() with seed 0 and a 128-wide projection."""
    cfg = dict(BERT_BASE, model_type="bert", hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0)
    return state_dict(cfg, BASE_P, 0), cfg


def bert_base_tokens():
    """(query tokens [16, 32], passage tokens [16, 256]) with BERT's special ids, padded to the longest of each side."""
    g = torch.Generator().manual_seed(1234)
    q = seq_tokens(g, BASE_PAIRS, BASE_SQ, BERT_BASE["vocab_size"], 0, lo=1000, cls_id=101, sep_id=102, min_len=4)
    d = seq_tokens(g, BASE_PAIRS, BASE_SD, BERT_BASE["vocab_size"], 0, lo=1000, cls_id=101, sep_id=102)
    return q, d


def sd_checksum(sd):
    return rerank_cases.sd_checksum(sd)
