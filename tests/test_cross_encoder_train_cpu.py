"""Cross-encoder training, the parts that need no GPU:

  * the training groups equal the reference DPRCrossAttentionTransform's (tests/golden/cross_train_groups.npz, made by
    tests/golden/make_golden_cross_train.py) in the train, eval and test stages, with sampled and truncated negatives,
    sampled positives, random negatives and the batch fill: each (question, passage) joined the reference's way
    reproduces its string, the labels are all 0 and the group size is the reference's;
  * the datamodule with use_cross_attention=True assembles the same groups on its background thread, tokenised as
    (question, passage) pairs; rows in the DPR retriever-output format and token-list passages are accepted;
  * the configs compose to the new task and datamodule classes;
  * num_labels=1 initialises a head on a head-less BERT / RoBERTa checkpoint (seeded), and num_labels=None still raises
    KeyError there;
  * group_ce refuses, with ValueError and before any GPU work, num_labels > 1, G < 2, G above the kernel's maximum, rows
    that are not whole groups, and attention / hidden dropout probabilities that differ.
"""
import json
import os
import sys

import numpy as np
import pytest
import torch

from tests import rerank_cases
from tests.util import GOLDEN

sys.path.insert(0, GOLDEN)
from make_golden_cross_train import CASES, batches  # noqa: E402


class _Pairs(torch.nn.Module):
    """Records what the transform would tokenise."""

    def forward(self, questions, passages):
        return {"questions": list(questions), "passages": list(passages)}


@pytest.mark.parametrize("case", sorted(CASES))
def test_groups_equal_reference_golden(case):
    from dpr_scale_b200.transforms.dpr_transform import DPRCrossAttentionTransform
    g = np.load(os.path.join(GOLDEN, "cross_train_groups.npz"))
    chunks, stage, seed, kw = batches(case)
    tf = DPRCrossAttentionTransform(_Pairs(), **kw)
    np.random.seed(seed)
    texts, labels, sizes = [], [], []
    for chunk in chunks:
        out = tf(chunk, stage)
        pairs = out["text_ids"]
        texts += [" ".join([q, tf.sep_token, p]) for q, p in zip(pairs["questions"], pairs["passages"])]
        labels += out["labels"].tolist()
        sizes.append(out["group_size"])
        assert out["labels"].dtype == torch.int64 and len(pairs["passages"]) == out["group_size"] * len(chunk)
    assert texts == g[f"{case}/text"].tolist()
    assert labels == g[f"{case}/label"].tolist() and set(labels) == {0}
    assert sizes == g[f"{case}/group_size"].tolist()


def test_short_rows_take_the_batch_fill():
    """Rows with fewer negatives than wanted are filled from the batch's positives and hard negatives."""
    from dpr_scale_b200.transforms.dpr_transform import DPRCrossAttentionTransform
    chunks, stage, seed, kw = batches("eval")
    rows = [json.loads(r) for r in chunks[0]]
    pool = {c["text"] if isinstance(c["text"], str) else " ".join(c["text"])
            for r in rows for c in r["positive_ctxs"] + r["hard_negative_ctxs"]}
    tf = DPRCrossAttentionTransform(_Pairs(), **kw)
    np.random.seed(seed)
    out = tf(chunks[0], "eval")
    G = out["group_size"]
    short = [i for i, r in enumerate(rows) if len(r["hard_negative_ctxs"]) < kw["num_val_negative"]]
    assert short
    for i in short:
        own = rows[i]["hard_negative_ctxs"]
        group = out["text_ids"]["passages"][i * G:(i + 1) * G]
        assert group[1:1 + len(own)] == [c["text"] for c in own]
        assert all(p in pool for p in group[1 + len(own):])


def test_retriever_output_rows_and_token_lists():
    from dpr_scale_b200.transforms.dpr_transform import DPRCrossAttentionTransform
    path = os.path.join(GOLDEN, "data", "synth.jsonl")
    lines = open(path, "rb").read().splitlines(keepends=True)
    tf = DPRCrossAttentionTransform(_Pairs(), num_negative=2)
    np.random.seed(0)
    out = tf([lines[4], lines[13], lines[14]], "train")
    assert out["group_size"] == 3 and out["labels"].tolist() == [0, 0, 0]
    passages = out["text_ids"]["passages"]
    assert all(isinstance(p, str) for p in passages)
    row13 = json.loads(lines[13])
    assert passages[3] == next(c["text"] for c in row13["ctxs"] if c["has_answer"])


@pytest.mark.parametrize("prefetch", [0, 2])
def test_datamodule_assembles_pair_tokenised_groups(tmp_path, prefetch):
    from dpr_scale_b200.datamodule.dpr import DenseRetrieverJsonlDataModule
    from dpr_scale_b200.transforms.hf_transform import HFTransform
    tf = HFTransform(rerank_cases.tokenizer_dir(str(tmp_path / "tok")), max_seq_len=64)
    path = str(tmp_path / "rows.jsonl")
    chunks, _, _, kw = batches("train")
    with open(path, "wb") as f:
        f.writelines(line for c in chunks for line in c)
    dm = DenseRetrieverJsonlDataModule(tf, path, path, path, batch_size=4, use_cross_attention=True,
                                       prefetch_batches=prefetch, device_prefetch=False, **kw)
    np.random.seed(11)
    got = list(dm.train_dataloader())
    np.random.seed(11)
    ref = DenseRetrieverJsonlDataModule(_Pairs(), path, path, path, batch_size=4, use_cross_attention=True,
                                        prefetch_batches=0, device_prefetch=False, **kw)
    want = list(ref.train_dataloader())
    assert len(got) == len(want) == 3
    for b, w in zip(got, want):
        enc = tf(w["text_ids"]["questions"], w["text_ids"]["passages"])
        for k in ("input_ids", "token_type_ids", "attention_mask"):
            assert torch.equal(b["text_ids"][k], enc[k])
        assert b["group_size"] == 4 and b["labels"].tolist() == [0] * 4
        assert int(b["text_ids"]["token_type_ids"].max()) == 1          # segment B: the passage


def test_bi_encoder_batches_unchanged_without_cross_attention(tmp_path):
    from dpr_scale_b200.datamodule.dpr import DenseRetrieverJsonlDataModule
    from dpr_scale_b200.transforms.dpr_transform import DPRTransform
    path = os.path.join(GOLDEN, "data", "synth.jsonl")
    dm = DenseRetrieverJsonlDataModule(_Pairs(), path, path, path)
    assert type(dm.dpr_transform) is DPRTransform


def test_configs_compose_to_the_training_classes():
    from dpr_scale_b200.utils.config import compose
    cfg = compose("config", ["task=cross_encoder_train", "task/model=cross_encoder", "datamodule=cross_encoder_train",
                             "task.model.model_path=/m", "+task.model.num_labels=1", "datamodule.train_path=a",
                             "datamodule.val_path=b", "datamodule.test_path=c"])
    assert cfg.task._target_ == "dpr_scale_b200.task.cross_encoder_train_task.CrossEncoderTrainTask"
    assert cfg.task.model._target_ == "dpr_scale_b200.models.citadel_models.cross_encoder.CrossEncoder"
    assert cfg.datamodule._target_ == "dpr_scale_b200.datamodule.dpr.DenseRetrieverJsonlDataModule"
    assert cfg.datamodule.use_cross_attention is True
    assert cfg.checkpoint_callback.monitor == "valid_mrr"
    from dpr_scale_b200.task.cross_encoder_task import CrossEncoderTask
    from dpr_scale_b200.task.cross_encoder_train_task import CrossEncoderTrainTask
    from dpr_scale_b200.utils.config import instantiate
    cfg.task.datamodule = None
    task = instantiate(cfg.task, _recursive_=False)
    assert isinstance(task, CrossEncoderTrainTask) and isinstance(task, CrossEncoderTask)


def _headless_dir(tmp_path, kind):
    """A plain BertModel / RobertaModel checkpoint: body weights only (BERT keeps its pooler)."""
    from transformers import BertConfig, BertModel, RobertaConfig, RobertaModel
    cfg = rerank_cases.tiny_config(kind)
    cfg.pop("num_labels")
    torch.manual_seed(5)
    model = BertModel(BertConfig(**cfg)) if kind == "bert" else RobertaModel(RobertaConfig(**cfg), add_pooling_layer=False)
    path = str(tmp_path / kind)
    model.save_pretrained(path)
    return path, model


@pytest.mark.parametrize("kind", ["bert", "roberta"])
def test_num_labels_initialises_a_missing_head(tmp_path, kind):
    from dpr_scale_b200.models.citadel_models.cross_encoder import CrossEncoder
    path, hf = _headless_dir(tmp_path, kind)
    with pytest.raises(KeyError):
        CrossEncoder(path)
    a, b = CrossEncoder(path, num_labels=1), CrossEncoder(path, num_labels=1)
    assert a.num_labels == 1
    dense, out = a._head_linears()
    assert out.weight.shape == (1, a.config["hidden_size"]) and bool((out.bias == 0).all())
    assert 0.01 < float(out.weight.std()) < 0.03                      # N(0, initializer_range = 0.02)
    for (k, x), (_, y) in zip(a.state_dict().items(), b.state_dict().items()):
        assert torch.equal(x, y), k                                    # seeded
    if kind == "bert":                                                 # the checkpoint's pooler is kept
        assert torch.equal(dense.weight, hf.pooler.dense.weight.detach())
    word = a.state_dict()[f"transformer.{a.body_name}.embeddings.word_embeddings.weight"]
    assert torch.equal(word, hf.embeddings.word_embeddings.weight.detach())


def test_num_labels_replaces_a_head_of_another_shape(tmp_path):
    from dpr_scale_b200.models.citadel_models.cross_encoder import CrossEncoder
    cfg = rerank_cases.tiny_config("roberta")                          # a 2-label head
    path = rerank_cases.hf_model_dir(str(tmp_path / "r"), cfg, 3)
    two = CrossEncoder(path)
    one = CrossEncoder(path, num_labels=1)
    assert two.num_labels == 2 and one.num_labels == 1
    assert torch.equal(one._head_linears()[0].weight, two._head_linears()[0].weight)   # same shape: loaded
    assert one._head_linears()[1].weight.shape == (1, cfg["hidden_size"])


def test_training_refusals_raise_before_gpu_work():
    from dpr_scale_b200 import ops
    from dpr_scale_b200.models.citadel_models.cross_encoder import CrossEncoder
    tokens = {"input_ids": torch.ones(8, 6, dtype=torch.int64)}
    two = CrossEncoder.from_config(rerank_cases.tiny_config("roberta")).train()
    with pytest.raises(ValueError, match="one relevance label"):
        two.group_ce(tokens, torch.zeros(2, dtype=torch.int64), 4)
    one = CrossEncoder.from_config(rerank_cases.tiny_config("bert")).train()
    for G in (1, 3, ops.SEQCLS_GROUP_MAX + 8):
        rows = {"input_ids": torch.ones(G * 2 if G != 3 else 8, 6, dtype=torch.int64)}
        with pytest.raises(ValueError):
            one.group_ce(rows, torch.zeros(2, dtype=torch.int64), G)
    cfg = dict(rerank_cases.tiny_config("bert"), hidden_dropout_prob=0.1, attention_probs_dropout_prob=0.2)
    with pytest.raises(ValueError, match="attention_probs_dropout_prob"):
        CrossEncoder.from_config(cfg).train().group_ce(tokens, torch.zeros(2, dtype=torch.int64), 4)


def test_dropout_probabilities_follow_the_config():
    from dpr_scale_b200.models.citadel_models.cross_encoder import CrossEncoder
    base = rerank_cases.tiny_config("bert")
    m = CrossEncoder.from_config(dict(base, hidden_dropout_prob=0.1, attention_probs_dropout_prob=0.1))
    assert (m.hidden_dropout, m.head_dropout, m._body.dropout) == (0.1, 0.1, 0.1)
    m = CrossEncoder.from_config(dict(base, hidden_dropout_prob=0.1, attention_probs_dropout_prob=0.1,
                                      classifier_dropout=0.3))
    assert m.head_dropout == 0.3
    assert not m._body.training
    m.train()
    assert m._body.training
    m.eval()
    assert not m._body.training
