"""Sequences of up to 512 tokens, without a GPU:

  * the oracle (oracle/hf_path.CLSEncoder + oracle/task) pinned to the UNMODIFIED reference at S = 512 on BERT-base
    (tests/golden/realdims_bert_base_s512.npz, made by tests/golden/make_golden_long.py): sequence 0 is 512 tokens
    long, so the last row of the position table is used;
  * HFEncoder rejects, before anything reaches the CUDA library, a batch whose position ids would fall outside the
    position table (BERT: S > max_position_embeddings; RoBERTa: S > max_position_embeddings - pad_token_id - 1,
    because its positions are pad-derived) or that is longer than 512 tokens.
"""
import pytest
import torch

from oracle import hf_path, task as otask
from tests import realdims, realdims_long
from tests.util import load_golden, rel_l2, sub

TINY = dict(vocab_size=64, hidden_size=128, num_hidden_layers=2, num_attention_heads=2, intermediate_size=256)


def test_oracle_matches_reference_golden_bert_base_s512():
    name = realdims_long.NAME
    kind, cfg, B, n, S, T = realdims.CASES[name]
    g = load_golden(f"realdims_{name}.npz")
    qm, cm = realdims.hf_models(kind, cfg)
    assert torch.equal(realdims.checksums(qm), g["sum_q"]) and torch.equal(realdims.checksums(cm), g["sum_c"])
    regen = realdims.batch(name)
    b = sub(g, "batch/")
    assert torch.equal(regen["contexts_ids"]["input_ids"], b["contexts_ids/input_ids"])
    assert torch.equal(regen["query_ids"]["input_ids"], b["query_ids/input_ids"])
    assert regen["query_ids"]["input_ids"].shape[1] == 512 and int(regen["query_ids"]["attention_mask"][0].sum()) == 512
    assert torch.equal(regen["ctx_mask"], b["ctx_mask"].bool()) and bool(regen["ctx_mask"].any())
    qe, ce = hf_path.CLSEncoder(None, model=qm), hf_path.CLSEncoder(None, model=cm)
    q, c = qe(regen["query_ids"]), ce(regen["contexts_ids"])
    assert rel_l2(q.detach(), g["q_emb"]) <= 1e-5 and rel_l2(c.detach(), g["c_emb"]) <= 1e-5
    loss, logits = otask.in_batch_loss(q, c, regen["ctx_mask"], regen["pos_ctx_indices"], T)
    fin = torch.isfinite(g["logits"])
    assert torch.equal(torch.isfinite(logits), fin)
    assert float((logits.detach()[fin] - g["logits"][fin]).abs().max()) <= 1e-3
    assert abs(float(loss) - float(g["loss"])) <= 1e-4
    loss.backward()
    for side, m in (("q", qm), ("c", cm)):
        params = dict(m.named_parameters())
        names = realdims.sampled_grad_names(cfg)
        # an analytically zero gradient (the context side's last LayerNorm bias) is fp32 noise whose digits depend on
        # the CPU's summation order: it must sit at the noise floor in both runs
        floor = 1e-6 * max(float(g[f"grad_{side}/{k}"].norm()) for k in names)
        for k in names:
            want = g[f"grad_{side}/{k}"]
            got = realdims.sample(k, params[k].grad)
            assert rel_l2(got, want) <= 1e-3 or max(float(want.norm()), float(got.norm())) < floor, (side, k, rel_l2(got, want))


def _encoder(kind, max_pos):
    from dpr_scale_b200.models.hf_model import HFEncoder
    cfg = dict(TINY, model_type=kind, max_position_embeddings=max_pos)
    if kind == "roberta":
        cfg.update(type_vocab_size=1, pad_token_id=1, layer_norm_eps=1e-5)
    return HFEncoder.from_config(cfg, dropout=0.0)


def _tokens(S, pad_id=0):
    ids = torch.randint(3, 64, (2, S), generator=torch.Generator().manual_seed(0))
    ids[ids == pad_id] = 5
    return {"input_ids": ids, "attention_mask": torch.ones(2, S, dtype=torch.long)}


@pytest.mark.parametrize("grad", [True, False])
def test_bert_rejects_positions_beyond_the_table(grad):
    enc = _encoder("bert", 512)
    with torch.set_grad_enabled(grad), pytest.raises(ValueError, match="max_position_embeddings"):
        enc(_tokens(513))
    with pytest.raises(ValueError, match="max_position_embeddings"):
        enc._prep_tokens(_tokens(513))
    enc._prep_tokens(_tokens(512))      # the whole table is usable


def test_roberta_rejects_pad_derived_positions_beyond_the_table():
    # positions run pad_id + 1 .. pad_id + S: S = 512 needs 514 rows
    enc = _encoder("roberta", 513)
    with pytest.raises(ValueError, match="max_position_embeddings"):
        enc(_tokens(512, pad_id=1))
    enc._prep_tokens(_tokens(511, pad_id=1))


def test_roberta_s512_passes_the_position_check():
    from dpr_scale_b200._lib import DprbError
    enc = _encoder("roberta", 514)
    _, _, pos, _, N, S = enc._prep_tokens(_tokens(512, pad_id=1))
    assert (N, S) == (2, 512) and int(pos.max()) == 513
    # the check passes; on a machine without the module on a GPU the call then stops at the CUDA-only error
    with pytest.raises(DprbError):
        enc(_tokens(512, pad_id=1))


def test_longer_than_512_is_rejected_even_with_a_larger_table():
    enc = _encoder("bert", 1024)
    with pytest.raises(ValueError, match="512"):
        enc(_tokens(600))
