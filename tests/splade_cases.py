"""Deterministic recipes shared by the SPLADE / dense-rerank goldens (tests/golden/make_golden_splade.py) and their
tests: tiny BERT / RoBERTa SPLADE encoders, a tiny HFEncoder with a projection, the rerank task's checkpoints and the
BERT-base-dims SPLADE encoder.  No weights are committed: every state dict is rebuilt from its seed here (same torch +
transformers => same RNG stream), and the goldens hold fp64 checksums that prove it is the one the reference ran.
Tokens, the fixture run and the datamodule settings are those of tests/colbert_cases.py and tests/rerank_cases.py."""
import torch

from tests import colbert_cases, multivec_cases, rerank_cases
from tests.realdims import BERT_BASE

# name: (encoder kind, seed)
TINY = {"splade_bert": ("bert", 51), "splade_roberta": ("roberta", 52)}
# the rerank task's encoders: name -> (model, encoder kind, HFEncoder projection, seed)
TASK = {"hf": ("hf", "bert", 64, 61), "splade": ("splade", "bert", None, 51)}
TARGETS = {"hf": "dpr_scale.models.hf_model.HFEncoder", "splade": "dpr_scale.models.citadel_models.splade_model.SPLADEEncoder"}
HF_PROJ = 64


def state_dict(kind, seed):
    """A SPLADEEncoder state dict: ``transformer.*`` of a seeded masked-LM model, the tied decoder included."""
    return multivec_cases.state_dict("citadel", colbert_cases.encoder_config(kind), None, None, seed)


def tiny_state_dict(name, seed_offset=0):
    kind, seed = TINY[name]
    return state_dict(kind, seed + seed_offset)


def hf_state_dict(seed):
    """An HFEncoder state dict: ``transformer.*`` of a seeded BertModel (pooler included) + the Linear + LayerNorm
    projection ``project.{0,1}.*``."""
    sd = colbert_cases.state_dict(colbert_cases.encoder_config("bert"), None, seed)
    g = torch.Generator().manual_seed(seed + 300)
    sd["project.0.weight"] = 0.05 * torch.randn(HF_PROJ, 128, generator=g)
    sd["project.0.bias"] = 0.02 * torch.randn(HF_PROJ, generator=g)
    sd["project.1.weight"] = 1.0 + 0.05 * torch.randn(HF_PROJ, generator=g)
    sd["project.1.bias"] = 0.02 * torch.randn(HF_PROJ, generator=g)
    return sd


def encoder_state_dict(model, seed):
    return hf_state_dict(seed) if model == "hf" else state_dict("bert", seed)


def task_state_dict(model):
    """The rerank task's checkpoint: two different encoders (query: the seed, context: the seed + 1000)."""
    _, _, _, seed = TASK[model]
    sd = {"query_encoder." + k: v for k, v in encoder_state_dict(model, seed).items()}
    sd.update({"context_encoder." + k: v for k, v in encoder_state_dict(model, seed + 1000).items()})
    return sd


def model_dir(path, model, seed):
    """A checkpoint directory the reference's and this repo's encoder both load (plus the fixture tokenizer)."""
    from transformers import BertConfig, BertModel
    cfg = colbert_cases.encoder_config("bert")
    if model == "hf":
        hf = BertModel(BertConfig(**cfg))
        hf.load_state_dict({k[len("transformer."):]: v for k, v in hf_state_dict(seed).items()
                            if k.startswith("transformer.")}, strict=False)
    else:
        hf, _ = multivec_cases.hf_masked_lm(cfg, seed)
    hf.save_pretrained(path)
    return rerank_cases.tokenizer_dir(path)


def tiny_model_dir(path, name):
    kind, seed = TINY[name]
    hf, _ = multivec_cases.hf_masked_lm(colbert_cases.encoder_config(kind), seed)
    hf.save_pretrained(path)
    return rerank_cases.tokenizer_dir(path)


def tiny_tokens(cfg, S=20, n=6, seed=19):
    """Padded random tokens; the last row has no valid token after token 0 (its SPLADE vector is 0)."""
    toks = colbert_cases.seq_tokens(torch.Generator().manual_seed(seed), n, S, cfg["vocab_size"], cfg["pad_token_id"])
    toks["attention_mask"][-1, 1:] = 0
    toks["input_ids"][-1, 1:] = cfg["pad_token_id"]
    return toks


def build(name, sd=None):
    """This repo's SPLADEEncoder of `name` (random init from the config), with `sd` loaded strictly when given."""
    from dpr_scale_b200.models.citadel_models.splade_model import SPLADEEncoder
    kind, _ = TINY[name]
    m = SPLADEEncoder.from_config(colbert_cases.encoder_config(kind))
    if sd is not None:
        m.load_state_dict(sd, strict=True)
    return m


def bert_base_state_dict():
    """(state dict, config): BERT-base dims, the SPLADE recipe with seed 0."""
    cfg = dict(BERT_BASE, model_type="bert", hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0)
    return multivec_cases.state_dict("citadel", cfg, None, None, 0), cfg


def bert_base_tokens():
    return colbert_cases.bert_base_tokens()


BASE_COL_STRIDE = 16    # the BERT-base golden keeps every 16th vocabulary column of the reps
