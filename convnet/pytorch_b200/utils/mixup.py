"""Input mixing regularisers with the interface of the reference's utils/mixup.py: ``MixUp`` and ``CutMix``.

    m.sample(alpha, batch_size)     draws the partner permutation (torch.randperm, CPU generator) and ONE lambda
                                    (numpy.random.beta(alpha, alpha)), in that order; stored as m.mix_index /
                                    m.mix_values (fp32 [1])
    m(x)                            the mixed batch (training mode only; identity otherwise)
    m.mix_target(y, n_class)        the soft target lambda*onehot(y) + (1-lambda)*onehot(y[perm])

MixUp:  x' = lambda*x + (1-lambda)*x[perm] in fp32, as two products and one sum.
CutMix: the centre of the box is drawn when the batch is mixed (numpy.random.randint(H), then randint(W)); rows
        [r0, r1) x columns [c0, c1) of every sample are replaced by those of its partner and lambda becomes the
        uncovered fraction of the image, 1 - box area / (H*W).  ``box`` keeps (r0, r1, c0, c1).

These modules are the only place that draws the mixing randomness.  The CPU / stock-torch path applies them to the
batch directly; the CUDA kernel path (Trainer with a converted model) reads ``mix_index``, ``mix_values`` and ``box``
and mixes inside the input relayout and loss kernels instead.  Per-sample lambdas (``sample_batch=True`` of the
reference) are not provided.
"""
import math

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F


class MixUp(nn.Module):
    def __init__(self, batch_dim=0):
        super(MixUp, self).__init__()
        self.batch_dim = batch_dim
        self.reset()

    def reset(self):
        self.enabled = False
        self.mix_values = None
        self.mix_index = None

    def mix(self, x1, x2):
        """lambda*x1 + (1-lambda)*x2 with lambda broadcast along the batch dimension."""
        view = [1] * x1.dim()
        view[self.batch_dim] = -1
        lam = self.mix_values.to(device=x1.device).view(*view)
        return lam * x1 + (1. - lam) * x2

    def sample(self, alpha, batch_size, sample_batch=False):
        if sample_batch:
            raise NotImplementedError('per-sample mixing values (sample_batch=True) are not supported')
        self.mix_index = torch.randperm(batch_size)
        self.mix_values = torch.tensor([np.random.beta(alpha, alpha)], dtype=torch.float)

    def _active(self):
        return self.training and self.mix_values is not None

    def mix_target(self, y, n_class):
        if not self._active():
            return y
        y = F.one_hot(y, n_class).to(dtype=torch.float)
        return self.mix(y, y.index_select(self.batch_dim, self.mix_index.to(device=y.device)))

    def forward(self, x):
        if not self._active():
            return x
        return self.mix(x, x.index_select(self.batch_dim, self.mix_index.to(device=x.device)))


class CutMix(MixUp):
    def reset(self):
        super(CutMix, self).reset()
        self.box = None

    def sample(self, alpha, batch_size, sample_batch=False):
        if sample_batch:
            raise NotImplementedError('CutMix draws one box per batch (sample_batch=True is not supported)')
        super(CutMix, self).sample(alpha, batch_size)

    def draw_box(self, H, W):
        """Draw the box for an H x W batch from the current lambda and replace lambda by the uncovered fraction.
        Returns (r0, r1, c0, c1).  The half-widths are int(H*sqrt(1-lambda))//2 and int(W*sqrt(1-lambda))//2 around a
        uniform centre, clipped to the image -- so a box at the border is smaller and lambda grows accordingly."""
        lam = float(self.mix_values)
        cut = math.sqrt(1. - lam)
        half_h, half_w = int(H * cut) // 2, int(W * cut) // 2
        cy = int(np.random.randint(H))
        cx = int(np.random.randint(W))
        r0, r1 = min(max(cy - half_h, 0), H), min(max(cy + half_h, 0), H)
        c0, c1 = min(max(cx - half_w, 0), W), min(max(cx + half_w, 0), W)
        self.box = (r0, r1, c0, c1)
        self.mix_values.fill_(1 - ((r1 - r0) * (c1 - c0) / (H * W)))
        return self.box

    def mix_image(self, x1, x2):
        """x1 with the box of x2 pasted in (x1 is modified in place, as in the reference)."""
        r0, r1, c0, c1 = self.draw_box(x1.size(-2), x1.size(-1))
        x1[..., r0:r1, c0:c1] = x2[..., r0:r1, c0:c1]
        return x1

    def forward(self, x):
        if not self._active():
            return x
        return self.mix_image(x, x.index_select(self.batch_dim, self.mix_index.to(device=x.device)))
