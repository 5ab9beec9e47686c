"""Deterministic recipes shared by the COIL / CITADEL goldens (tests/golden/make_golden_multivec.py) and their tests:
tiny BERT / RoBERTa COIL and CITADEL encoders, the rerank task's checkpoint and the BERT-base-dims encoders.  No weights
are committed: every state dict is rebuilt from its seed here (same torch + transformers => same RNG stream), and the
goldens hold fp64 checksums that prove it is the one the reference ran.  Tokens, the fixture run and the datamodule
settings are those of tests/colbert_cases.py and tests/rerank_cases.py."""
import torch

from tests import colbert_cases, rerank_cases
from tests.realdims import BERT_BASE

# name: (model, encoder kind, token projection, CLS projection, seed)
TINY = {"coil_bert": ("coil", "bert", 64, 32, 41), "coil_roberta": ("coil", "roberta", 64, None, 42),
        "citadel_bert": ("citadel", "bert", 32, 64, 43), "citadel_roberta": ("citadel", "roberta", None, 64, 44)}
POOLS = ("sum", "max")
TASK_TOPK = (2, 1)                                  # (query_topk, context_topk) of the task runs
BASE_PAIRS, BASE_SQ, BASE_SD = 16, 32, 256
BASE = {"coil": (128, 128), "citadel": (32, 128)}   # (token projection, CLS projection), the reference's configs
TARGETS = {"coil": "coil_model.COILEncoder", "citadel": "citadel_model.CITADELEncoder"}


def ctor_kwargs(model, proj, cls_proj):
    """The encoder's constructor keywords (the reference's names)."""
    if model == "coil":
        return {"projection_dim": proj, "cls_projection_dim": cls_proj}
    return {"tok_projection_dim": proj, "cls_projection_dim": cls_proj}


def _perturb(model, seed):
    g = torch.Generator().manual_seed(seed + 100)
    with torch.no_grad():
        for name, p in model.named_parameters():
            if name.endswith("bias"):
                p.copy_(0.02 * torch.randn(p.shape, generator=g))
            elif "LayerNorm.weight" in name or "layer_norm.weight" in name:
                p.copy_(1.0 + 0.02 * torch.randn(p.shape, generator=g))
    return g


def hf_masked_lm(cfg, seed):
    """A seeded HF BertForMaskedLM / RobertaForMaskedLM (HF init, then non-trivial biases and LayerNorm affines)."""
    from transformers import BertConfig, BertForMaskedLM, RobertaConfig, RobertaForMaskedLM
    torch.manual_seed(seed)
    model = BertForMaskedLM(BertConfig(**cfg)) if cfg["model_type"] == "bert" else RobertaForMaskedLM(RobertaConfig(**cfg))
    return model, _perturb(model, seed)


def state_dict(model, cfg, proj, cls_proj, seed):
    """A COILEncoder / CITADELEncoder state dict with the reference's keys: COIL = colbert_cases.state_dict (body with
    its pooler + ``project.0.*``) + ``cls_project.0.*``; CITADEL = ``transformer.*`` of a seeded masked-LM model (the
    tied decoder included) + ``cls_project.0.*`` + ``tok_project.0.*``."""
    H = cfg["hidden_size"]
    if model == "coil":
        sd = colbert_cases.state_dict(cfg, proj, seed)
        g = torch.Generator().manual_seed(seed + 200)
        if cls_proj:
            sd["cls_project.0.weight"] = 0.05 * torch.randn(cls_proj, H, generator=g)
            sd["cls_project.0.bias"] = 0.02 * torch.randn(cls_proj, generator=g)
        return sd
    lm, g = hf_masked_lm(cfg, seed)
    sd = {"transformer." + k: v.detach().clone() for k, v in lm.state_dict().items()
          if not k.endswith(("position_ids", "token_type_ids"))}
    for key, dim in (("cls_project", cls_proj), ("tok_project", proj)):
        if dim:
            sd[f"{key}.0.weight"] = 0.05 * torch.randn(dim, H, generator=g)
            sd[f"{key}.0.bias"] = 0.02 * torch.randn(dim, generator=g)
    return sd


def tiny_state_dict(name, seed_offset=0):
    model, kind, proj, cls_proj, seed = TINY[name]
    return state_dict(model, colbert_cases.encoder_config(kind), proj, cls_proj, seed + seed_offset)


def task_state_dict(name):
    """The rerank task's checkpoint: two different encoders of `name` (query: its seed, context: the seed + 1000)."""
    sd = {"query_encoder." + k: v for k, v in tiny_state_dict(name).items()}
    sd.update({"context_encoder." + k: v for k, v in tiny_state_dict(name, 1000).items()})
    return sd


def model_dir(path, name):
    """A checkpoint directory the reference's and this repo's encoder both load (plus the fixture tokenizer)."""
    from transformers import BertConfig, BertModel, RobertaConfig, RobertaModel
    model, kind, _, _, seed = TINY[name]
    cfg = colbert_cases.encoder_config(kind)
    body = {k[len("transformer."):]: v for k, v in tiny_state_dict(name).items() if k.startswith("transformer.")}
    if model == "coil":
        hf = BertModel(BertConfig(**cfg)) if kind == "bert" else RobertaModel(RobertaConfig(**cfg))
    else:
        hf, _ = hf_masked_lm(cfg, seed)
    hf.load_state_dict(body, strict=False)
    hf.save_pretrained(path)
    return rerank_cases.tokenizer_dir(path)


def build(name, sd=None):
    """This repo's encoder of `name` (random init from the config), with `sd` loaded strictly when given."""
    from dpr_scale_b200.models.citadel_models.citadel_model import CITADELEncoder
    from dpr_scale_b200.models.citadel_models.coil_model import COILEncoder
    model, kind, proj, cls_proj, _ = TINY[name]
    cls = COILEncoder if model == "coil" else CITADELEncoder
    m = cls.from_config(colbert_cases.encoder_config(kind), proj, cls_proj)
    if sd is not None:
        m.load_state_dict(sd, strict=True)
    return m


def bert_base_state_dict(model):
    """(state dict, config): BERT-base dims, the recipe of state_dict() with seed 0 and the reference config's
    projections."""
    cfg = dict(BERT_BASE, model_type="bert", hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0)
    proj, cls_proj = BASE[model]
    return state_dict(model, cfg, proj, cls_proj, 0), cfg


def bert_base_tokens():
    return colbert_cases.bert_base_tokens()
