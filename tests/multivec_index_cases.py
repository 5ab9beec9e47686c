"""Deterministic recipes shared by the multi-vector index goldens (tests/golden/make_golden_multivec_index.py) and
their tests: which tiny COIL / CITADEL encoder (tests/multivec_cases.py) runs with which task keywords, and the two
token batches each case encodes.  The second batch has a passage whose only unmasked token is token 0."""
import torch

from tests import colbert_cases, multivec_cases

# passage cases: name -> (encoder, topk, add_cls, add_context_id, weight_threshold)
PASSAGE = {"coil_bert": ("coil_bert", 1, False, False, 0.0), "coil_bert_cls": ("coil_bert", 1, True, False, 0.0),
           "coil_roberta": ("coil_roberta", 1, False, False, 0.0),
           "citadel_bert_k1": ("citadel_bert", 1, True, False, 0.0),
           "citadel_bert_k2": ("citadel_bert", 2, False, False, 0.0),
           "citadel_bert_k2_thr": ("citadel_bert", 2, False, False, 0.4),
           "citadel_bert_k2_ctx": ("citadel_bert", 2, False, True, 0.0),
           "citadel_roberta_k2": ("citadel_roberta", 2, True, False, 0.0)}
# query cases: name -> (encoder, topk, add_cls)
QUERY = {"coil_bert": ("coil_bert", 1, True), "citadel_bert_k2": ("citadel_bert", 2, True),
         "citadel_roberta_k1": ("citadel_roberta", 1, False)}
SHAPES = ((4, 12), (3, 16))          # (sequences, tokens) of the two batches


def batches(encoder, seed=5):
    """[(tokens, ids)]: two padded random token batches for `encoder`; ids are corpus ids (passages) or topic ids."""
    kind = multivec_cases.TINY[encoder][1]
    cfg = colbert_cases.encoder_config(kind)
    g = torch.Generator().manual_seed(seed)
    out, first = [], 100
    for b, (n, S) in enumerate(SHAPES):
        toks = colbert_cases.seq_tokens(g, n, S, cfg["vocab_size"], cfg["pad_token_id"])
        if b == 1:                                    # token 0 alone
            toks["attention_mask"][1] = 0
            toks["attention_mask"][1, 0] = 1
            toks["input_ids"][1, 1:] = cfg["pad_token_id"]
        out.append((toks, [str(first + i) for i in range(n)]))
        first += n
    return out


def task_kwargs(encoder, model_dir, topk, add_cls):
    """Keywords both tasks (the reference's and this repo's) take, with the model config for `encoder`."""
    model, kind, proj, cls_proj, _ = multivec_cases.TINY[encoder]
    return dict(add_cls=add_cls, query_topk=topk, context_topk=topk, transform={}, datamodule=None, optim={},
                shared_model=False, in_batch_eval=False,
                model=dict({"model_path": model_dir, "dropout": 0.1}, **multivec_cases.ctor_kwargs(model, proj, cls_proj)))
