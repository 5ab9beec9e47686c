"""Deterministic recipes shared by the cross-encoder goldens (tests/golden/make_golden_rerank.py) and their tests: the
fixture run, tokenizer and datamodule settings, the tiny BERT / RoBERTa sequence classifiers, pair tokens, and the
BERT-base-dims classifier.  No weights are committed: every model is rebuilt from its seed here (same torch +
transformers => same RNG stream), and the goldens hold fp64 checksums that prove it is the one the reference ran."""
import os

import torch

from tests.realdims import BERT_BASE, checksums  # noqa: F401

DATA = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "data")
MAX_LEN = 24
VOCAB = len(open(os.path.join(DATA, "vocab.txt")).read().split())

TINY_BASE = dict(vocab_size=VOCAB, hidden_size=128, num_hidden_layers=2, num_attention_heads=2, intermediate_size=256,
                 hidden_act="gelu", hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0, type_vocab_size=2)
TINY = {
    "bert": dict(seed=21, config=dict(TINY_BASE, model_type="bert", max_position_embeddings=512, pad_token_id=0,
                                      layer_norm_eps=1e-12, num_labels=1)),
    # type_vocab_size 2 because the fixture tokenizer is a BERT one: pairs carry segment-B token types
    "roberta": dict(seed=22, config=dict(TINY_BASE, model_type="roberta", max_position_embeddings=514, pad_token_id=1,
                                         layer_norm_eps=1e-5, num_labels=2)),
}
ORACLE_CFG = {"bert": {"layers": 2, "heads": 2, "ln_eps": 1e-12, "pad_id": 0, "roberta": False},
              "roberta": {"layers": 2, "heads": 2, "ln_eps": 1e-5, "pad_id": 1, "roberta": True}}
BASE_PAIRS, BASE_S = 16, 256


def tiny_config(kind):
    return dict(TINY[kind]["config"])


def datamodule_kwargs():
    return dict(test_path=os.path.join(DATA, "rerank_run.trec"), test_question_path=os.path.join(DATA, "questions.tsv"),
                test_passage_path=os.path.join(DATA, "passages.tsv"), test_batch_size=5, use_title=True)


def tokenizer_dir(path):
    """A BERT WordPiece tokenizer over the fixture vocabulary (vocab.txt + tokenizer_config.json naming the class, so
    that a RoBERTa model directory gets it too; a config.json only where the directory has none)."""
    import json
    from transformers import BertConfig
    os.makedirs(path, exist_ok=True)
    if not os.path.exists(os.path.join(path, "config.json")):
        BertConfig(vocab_size=VOCAB, hidden_size=16, num_hidden_layers=1, num_attention_heads=1,
                   intermediate_size=16).save_pretrained(path)
    with open(os.path.join(DATA, "vocab.txt")) as s, open(os.path.join(path, "vocab.txt"), "w") as d:
        d.write(s.read())
    with open(os.path.join(path, "tokenizer_config.json"), "w") as f:
        json.dump({"tokenizer_class": "BertTokenizer", "do_lower_case": True}, f)
    return path


def hf_model(cfg, seed):
    """HF ...ForSequenceClassification with HF init, then non-trivial biases and LayerNorm affines."""
    from transformers import BertConfig, BertForSequenceClassification, RobertaConfig, RobertaForSequenceClassification
    torch.manual_seed(seed)
    if cfg["model_type"] == "bert":
        model = BertForSequenceClassification(BertConfig(**cfg))
    else:
        model = RobertaForSequenceClassification(RobertaConfig(**cfg))
    g = torch.Generator().manual_seed(seed + 100)
    with torch.no_grad():
        for name, p in model.named_parameters():
            if name.endswith("bias"):
                p.copy_(0.02 * torch.randn(p.shape, generator=g))
            elif "LayerNorm.weight" in name:
                p.copy_(1.0 + 0.02 * torch.randn(p.shape, generator=g))
    return model.eval()


def hf_model_dir(path, cfg, seed):
    """A checkpoint directory the reference's and this repo's CrossEncoder both load (plus the fixture tokenizer)."""
    hf_model(cfg, seed).save_pretrained(path)
    return tokenizer_dir(path)


def reference_state_dict(kind):
    """The state_dict of the reference's CrossEncoder around the seeded tiny model of `kind` (``transformer.`` + the HF
    names), rebuilt from the seed."""
    model = hf_model(tiny_config(kind), TINY[kind]["seed"])
    return {"transformer." + k: v.detach().clone() for k, v in model.state_dict().items()}


def sd_checksum(sd):
    """Order-sensitive fp64 fingerprint of a state dict (tests/realdims.checksums over a dict)."""
    tot, wtot, n = 0.0, 0.0, 0
    for i, (k, p) in enumerate(sorted(sd.items())):
        if not p.dtype.is_floating_point:
            continue
        d = p.double()
        tot += float(d.sum())
        wtot += float((d.flatten()[::97] * (1 + (i % 7))).sum())
        n += p.numel()
    return torch.tensor([tot, wtot, float(n)], dtype=torch.float64)


def pair_tokens(gen, n, S, vocab, pad_id, lo=5, cls_id=2, sep_id=3):
    """[CLS] a [SEP] b [SEP] pad..., token types 1 on segment b; row 0 is full length, the others ~ U{S/3..S}."""
    lens = torch.randint(max(5, S // 3), S + 1, (n,), generator=gen)
    lens[0] = S
    ids = torch.randint(lo, vocab, (n, S), generator=gen)
    tt = torch.zeros(n, S, dtype=torch.long)
    for i in range(n):
        L = int(lens[i])
        a = int(torch.randint(1, L - 3, (1,), generator=gen))       # position of the first [SEP]
        ids[i, 0], ids[i, a], ids[i, L - 1] = cls_id, sep_id, sep_id
        tt[i, a + 1:L] = 1
    am = (torch.arange(S).unsqueeze(0) < lens.unsqueeze(1)).long()
    ids = ids * am + pad_id * (1 - am)
    return {"input_ids": ids, "token_type_ids": tt * am, "attention_mask": am}


def bert_base_seqcls():
    """(model, config): torch.manual_seed(0); BertForSequenceClassification(num_labels=1) at BERT-base dims, biases
    moved off zero with a second seeded generator."""
    from transformers import BertConfig, BertForSequenceClassification
    cfg = dict(BERT_BASE, model_type="bert", num_labels=1, hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0)
    torch.manual_seed(0)
    model = BertForSequenceClassification(BertConfig(**cfg))
    g = torch.Generator().manual_seed(1)
    with torch.no_grad():
        for name, p in model.named_parameters():
            if name.endswith("bias"):
                p.add_(0.02 * torch.randn(p.shape, generator=g))
    return model.eval(), cfg
