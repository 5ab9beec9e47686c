"""Shared inputs of the distillation / DrBoost goldens (tests/golden/make_golden_distill.py) and the tests that compare
against them: the tiny BERT configs, encoder weights drawn from a seeded generator (so the golden file stores outputs,
not state dicts) and the gradients the golden keeps."""
import torch

# the tiny BERT of the distillation task (make_golden.make_model_dir("bert", ...) has the same shape)
CFG = dict(vocab_size=64, hidden_size=128, num_hidden_layers=2, num_attention_heads=2, intermediate_size=256,
           max_position_embeddings=40)
# the weak DrBoost encoders: one layer
WEAK_CFG = dict(CFG, num_hidden_layers=1)
TASK_SEED = 21
# weak encoder i: (shared_model, projection_dim, query-encoder seed, context-encoder seed)
WEAK = [(False, None, 500, 501), (True, 16, 502, 503)]


def encoder_state(config, seed, projection_dim=None):
    """A state dict for HFEncoder (keys ``transformer.*`` / ``project.*``, the reference HFEncoder's names): every
    tensor 0.02 * N(0, 1) from a generator seeded with ``seed``, LayerNorm weights around 1; keys in sorted order."""
    from dpr_scale_b200.models.hf_model import HFEncoder
    shapes = {k: v.shape for k, v in
              HFEncoder.from_config(config, dropout=0.0, projection_dim=projection_dim).state_dict().items()}
    g = torch.Generator().manual_seed(seed)
    out = {}
    for k in sorted(shapes):
        x = 0.02 * torch.randn(shapes[k], generator=g)
        if k.endswith("LayerNorm.weight") or k == "project.1.weight":
            x += 1.0
        out[k] = x
    return out


def kept_gradient(name, numel):
    """The gradients the golden keeps: every tensor of at most 8192 values (biases, LayerNorms, the tiny embedding
    tables) and two weight matrices."""
    return numel <= 8192 or name in ("transformer.encoder.layer.1.attention.output.dense.weight",
                                     "transformer.encoder.layer.0.intermediate.dense.weight")
