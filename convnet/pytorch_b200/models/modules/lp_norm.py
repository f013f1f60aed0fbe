"""L1 batch normalization ("Norm matters: efficient and accurate normalization schemes in deep networks", Hoffer et al.
2018), the layer the reference's ``resnet(bn_norm='L1')`` builds (models/modules/lp_norm.py:238-291).

Per channel over the N*H*W values of a batch: mu = mean(x), L = mean|x - mu|, and the variance-free scale
s = 1 / (L * sqrt(pi/2) + eps) -- for a normal x, sqrt(pi/2) * E|x - mu| is its standard deviation.  The output is
(x - mu) * s * weight + bias.  In eval mode mu and s are the running buffers.

State, as the reference's layer keeps it:
  * ``running_var`` holds the running SCALE s, not a variance;
  * the momentum weights the OLD value: running = running * momentum + batch * (1 - momentum), so with the default
    0.1 a new batch counts 0.9; both buffers start at zero, so an untrained model in eval mode outputs ``bias``;
  * ``state_dict`` order is ``bias, weight, running_mean, running_var`` (no ``num_batches_tracked``), and ``bias`` is
    the first parameter.

The torch forward below is what runs on the CPU; a model converted with ``engine.convert_b200`` runs the kernels of
csrc/bn_l1.cu instead.
"""
import math

import torch
import torch.nn as nn

L1_FIX = math.sqrt(math.pi / 2)


class L1BatchNorm2d(nn.Module):
    affine = True
    track_running_stats = True

    def __init__(self, num_features, eps=1e-5, momentum=0.1):
        super(L1BatchNorm2d, self).__init__()
        self.num_features = num_features
        self.eps = eps
        self.momentum = momentum
        self.bias = nn.Parameter(torch.zeros(num_features))
        self.weight = nn.Parameter(torch.ones(num_features))
        self.register_buffer('running_mean', torch.zeros(num_features))
        self.register_buffer('running_var', torch.zeros(num_features))

    def extra_repr(self):
        return '{num_features}, eps={eps}, momentum={momentum}'.format(**self.__dict__)

    def forward(self, x):
        if self.training:
            mean = x.mean((0, 2, 3))
            scale = 1.0 / ((x - mean[None, :, None, None]).abs().mean((0, 2, 3)) * L1_FIX + self.eps)
            with torch.no_grad():
                m = self.momentum
                self.running_mean.mul_(m).add_(mean.detach().to(self.running_mean.dtype) * (1 - m))
                self.running_var.mul_(m).add_(scale.detach().to(self.running_var.dtype) * (1 - m))
        else:
            mean, scale = self.running_mean.to(x.dtype), self.running_var.to(x.dtype)
        out = (x - mean[None, :, None, None]) * scale[None, :, None, None]
        return out * self.weight[None, :, None, None] + self.bias[None, :, None, None]
