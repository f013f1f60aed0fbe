"""Activation checkpointing of a residual stage (``checkpoint_segments`` of ResNet_imagenet, the reference's
models/modules/checkpoint.py).  The wrapped stage is ``.module``, so state_dict keys gain ``.module.``
(``layer1.module.0.conv1.weight``) exactly as in the reference's checkpoints.

On the CPU the forward is torch.utils.checkpoint with the reentrant variant, the reference's behaviour: a checkpointed
segment runs under no_grad in the forward pass and again, in training mode, in the backward pass -- so every BatchNorm
inside it updates its running statistics twice per step.  With ``num_segments = k > 1`` the stage's
``len // k`` -block segments are checkpointed ``k - 1`` times and the remaining blocks run normally
(torch.utils.checkpoint.checkpoint_sequential).  A model converted with ``engine.convert_b200`` reads
``num_segments`` and recomputes the same segments in its own backward pass instead.
"""
import torch.nn as nn
from torch.utils.checkpoint import checkpoint, checkpoint_sequential


class CheckpointModule(nn.Module):
    def __init__(self, module, num_segments=1):
        super(CheckpointModule, self).__init__()
        if num_segments != 1 and not isinstance(module, nn.Sequential):
            raise ValueError('CheckpointModule: %d segments need an nn.Sequential' % num_segments)
        self.module = module
        self.num_segments = num_segments

    def segments(self):
        """[start, end) block ranges of ``.module`` that are recomputed in the backward pass."""
        if self.num_segments == 1:
            return [(0, len(self.module))]
        size = len(self.module) // self.num_segments
        return [(j * size, (j + 1) * size) for j in range(self.num_segments - 1)]

    def forward(self, x):
        if self.num_segments > 1:
            return checkpoint_sequential(self.module, self.num_segments, x, use_reentrant=True)
        return checkpoint(self.module, x, use_reentrant=True)
