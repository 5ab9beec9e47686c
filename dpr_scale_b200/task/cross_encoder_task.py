"""CrossEncoderTask — drop-in for ``dpr_scale.task.cross_encoder_task.CrossEncoderTask``
(/root/reference/dpr_scale/task/cross_encoder_task.py): same constructor keywords and hooks.  Inference only, as in the
reference: ``configure_optimizers`` builds nothing and there is no training step.  The model is the configured
cross-encoder (``dpr_scale_b200.models.citadel_models.cross_encoder.CrossEncoder``).
"""
import torch

from ..utils.config import instantiate
from ..utils.lightning_shim import LightningModule


class CrossEncoderTask(LightningModule):
    def __init__(
        self,
        transform,
        model,
        datamodule,
        optim,
        k=1,
        shared_model: bool = True,
        in_batch_eval: bool = True,
        warmup_steps: int = 0,
        fp16_grads: bool = False,
        pretrained_checkpoint_path: str = "",
    ):
        super().__init__()
        self.save_hyperparameters()
        self.transform_conf = transform.text_transform if hasattr(transform, "text_transform") else transform
        self.model_conf = model
        self.k = k
        self.fp16_grads = fp16_grads
        self.pretrained_checkpoint_path = pretrained_checkpoint_path
        self.setup_done = False

    def setup(self, stage: str):
        # a second setup("test") must not rebuild the model (that would drop a loaded state dict)
        if stage == "test" and self.setup_done:
            return
        self.call_configure_sharded_model_hook = False
        self.cross_encoder = instantiate(self.model_conf)
        if self.pretrained_checkpoint_path:
            ckpt = torch.load(self.pretrained_checkpoint_path, map_location="cpu", weights_only=False)
            self.load_state_dict(ckpt["state_dict"])
            print(f"Loaded state dict from {self.pretrained_checkpoint_path}")
        self.setup_done = True

    def on_load_checkpoint(self, checkpoint) -> None:
        self.setup("fit")

    def on_pretrain_routine_start(self):
        # the reference registers fp16_compress_hook for a training it does not implement; nothing to reduce here
        pass

    def configure_optimizers(self):
        pass

    def forward(self, token_ids):
        return self.cross_encoder(token_ids)
