"""ResNet family (CIFAR and ImageNet variants) on the reference's factory contract.

Public surface kept from the reference (models/resnet.py): ``resnet(**config)`` factory keyed by
``dataset`` / ``depth``; module attribute names (``conv1, bn1, layer1..4, fc``; blocks ``conv1..3, bn1..3,
downsample``) so that ``state_dict`` keys and shapes are interchangeable; per-model ``regime`` lists,
``sampled_data_regime`` / ``data_eval_regime`` for the Mix&Match size regimes; He-normal init with the
last BN of each residual branch zeroed (models/resnet.py:16-31).

The modules are ordinary ``torch.nn`` layers, which is what runs in the CPU configuration.  On a B200
the tree is handed to ``engine.convert_b200(model)``: parameters move into flat arenas and ``forward``
is served by the fused kernel pipeline; the ``nn`` layers then only name the parameters.
"""
import math

import torch
import torch.nn as nn

from .modules.checkpoint import CheckpointModule
from .modules.lp_norm import L1BatchNorm2d

__all__ = ['resnet', 'resnet_se']


_BN_TYPES = (nn.BatchNorm2d, L1BatchNorm2d)
_NORM_LAYERS = {None: nn.BatchNorm2d, 'L1': L1BatchNorm2d}    # model-config 'bn_norm'


def init_model(model):
    """He-normal conv weights (fan-out), BN gamma=1/beta=0, zero-init of each block's last BN gamma,
    fc ~ N(0, 0.01) with zero bias -- the reference's scheme (models/resnet.py:16-31), same RNG order.  L1 BN layers
    count as BN (the reference sees them through its rebinding of nn.BatchNorm2d)."""
    for m in model.modules():
        if isinstance(m, nn.Conv2d):
            fan_out = m.kernel_size[0] * m.kernel_size[1] * m.out_channels
            m.weight.data.normal_(0, math.sqrt(2. / fan_out))
        elif isinstance(m, _BN_TYPES):
            m.weight.data.fill_(1)
            m.bias.data.zero_()
    for m in model.modules():
        if isinstance(m, Bottleneck):
            nn.init.constant_(m.bn3.weight, 0)
        elif isinstance(m, BasicBlock):
            nn.init.constant_(m.bn2.weight, 0)
    model.fc.weight.data.normal_(0, 0.01)
    model.fc.bias.data.zero_()


def weight_decay_config(value=1e-4, log=False):
    """WeightDecay regularizer on everything that is neither a bias nor inside a BatchNorm."""
    return {'name': 'WeightDecay', 'value': value, 'log': log,
            'filter': {'parameter_name': lambda n: not n.endswith('bias'),
                       'module': lambda m: not isinstance(m, _BN_TYPES)}}


def mixsize_config(sz, base_size, base_batch, base_duplicates, adapt_batch, adapt_duplicates):
    """Batch size / duplicates for input size ``sz`` such that the per-step work stays comparable to the base
    configuration (Mix&Match, models/resnet.py:43-67)."""
    assert adapt_batch or adapt_duplicates or sz == base_size
    ratio = base_size / sz
    scale = ratio if (adapt_batch and adapt_duplicates) else ratio ** 2
    if scale * base_duplicates < 0.5:  # cannot go below one duplicate: adapt the batch instead
        adapt_duplicates, adapt_batch = False, True
    batch_size = int(round(scale * base_batch)) if adapt_batch else base_batch
    duplicates = int(round(scale * base_duplicates)) if adapt_duplicates else base_duplicates
    return {'input_size': sz, 'batch_size': batch_size, 'duplicates': max(1, duplicates)}


def linear_scale(lr0, lrT, T, t0=0):
    slope = (lrT - lr0) / T
    return "lambda t: {'lr': max(%s + (t - %s) * %s, 0)}" % (lr0, t0, slope)


def conv3x3(in_planes, out_planes, stride=1, groups=1, bias=False):
    return nn.Conv2d(in_planes, out_planes, kernel_size=3, stride=stride, padding=1, groups=groups, bias=bias)


class BasicBlock(nn.Module):
    """3x3 -> BN -> ReLU -> 3x3 -> BN, plus skip, ReLU."""

    def __init__(self, inplanes, planes, stride=1, expansion=1, downsample=None, groups=1,
                 residual_block=None, dropout=0., norm_layer=nn.BatchNorm2d):
        super(BasicBlock, self).__init__()
        self.conv1 = conv3x3(inplanes, planes, stride, groups=groups)
        self.bn1 = norm_layer(planes)
        self.relu = nn.ReLU(inplace=True)
        self.conv2 = conv3x3(planes, expansion * planes, groups=groups)
        self.bn2 = norm_layer(expansion * planes)
        self.downsample = downsample
        self.residual_block = residual_block
        self.stride = stride
        self.expansion = expansion
        self.dropout = nn.Dropout(dropout or 0)

    def forward(self, x):
        skip = x if self.downsample is None else self.downsample(x)
        if self.residual_block is not None:
            skip = self.residual_block(skip)
        out = self.dropout(self.relu(self.bn1(self.conv1(x))))
        out = self.bn2(self.conv2(out))
        return self.relu(out + skip)


class Bottleneck(nn.Module):
    """1x1 -> 3x3 (carries the stride, 'v1.5') -> 1x1 with BN/ReLU in between, plus skip, ReLU."""

    def __init__(self, inplanes, planes, stride=1, expansion=4, downsample=None, groups=1,
                 residual_block=None, dropout=0., norm_layer=nn.BatchNorm2d):
        super(Bottleneck, self).__init__()
        self.conv1 = nn.Conv2d(inplanes, planes, kernel_size=1, bias=False)
        self.bn1 = norm_layer(planes)
        self.conv2 = conv3x3(planes, planes, stride=stride, groups=groups)
        self.bn2 = norm_layer(planes)
        self.conv3 = nn.Conv2d(planes, planes * expansion, kernel_size=1, bias=False)
        self.bn3 = norm_layer(planes * expansion)
        self.relu = nn.ReLU(inplace=True)
        self.dropout = nn.Dropout(dropout or 0)
        self.downsample = downsample
        self.residual_block = residual_block
        self.stride = stride
        self.expansion = expansion

    def forward(self, x):
        skip = x if self.downsample is None else self.downsample(x)
        if self.residual_block is not None:
            skip = self.residual_block(skip)
        out = self.dropout(self.relu(self.bn1(self.conv1(x))))
        out = self.dropout(self.relu(self.bn2(self.conv2(out))))
        out = self.bn3(self.conv3(out))
        return self.relu(out + skip)


class ResNet(nn.Module):
    _b200 = None  # set by engine.convert_b200
    norm_layer = nn.BatchNorm2d   # class of every BN of the network (the constructors set it: L1BatchNorm2d for bn_norm='L1')

    def _make_layer(self, block, planes, blocks, expansion=1, stride=1, groups=1, residual_block=None,
                    dropout=None, mixup=False):
        if mixup:
            raise NotImplementedError('intermediate MixUp layers are outside the B200 hot path (SURVEY 2, #18)')
        out_planes = planes * expansion
        downsample = None
        if stride != 1 or self.inplanes != out_planes:
            downsample = nn.Sequential(
                nn.Conv2d(self.inplanes, out_planes, kernel_size=1, stride=stride, bias=False),
                self.norm_layer(out_planes))
        if residual_block is not None:
            residual_block = residual_block(out_planes)
        stages = [block(self.inplanes, planes, stride, expansion=expansion, downsample=downsample, groups=groups,
                        residual_block=residual_block, dropout=dropout, norm_layer=self.norm_layer)]
        self.inplanes = out_planes
        for _ in range(1, blocks):
            stages.append(block(self.inplanes, planes, expansion=expansion, groups=groups,
                                residual_block=residual_block, dropout=dropout, norm_layer=self.norm_layer))
        return nn.Sequential(*stages)

    def features(self, x):
        x = self.maxpool(self.relu(self.bn1(self.conv1(x))))
        x = self.layer4(self.layer3(self.layer2(self.layer1(x))))
        return self.avgpool(x).flatten(1)

    def forward(self, x):
        if self._b200 is not None:
            return self._b200.forward(x)
        return self.fc(self.features(x))


class ResNet_imagenet(ResNet):
    num_train_images = 1281167

    def __init__(self, num_classes=1000, inplanes=64, block=Bottleneck, residual_block=None,
                 layers=[3, 4, 23, 3], width=[64, 128, 256, 512], expansion=4, groups=[1, 1, 1, 1],
                 regime='normal', scale_lr=1, ramp_up_lr=True, ramp_up_epochs=5, checkpoint_segments=0,
                 mixup=False, epochs=90, base_devices=4, base_device_batch=64, base_duplicates=1,
                 base_image_size=224, mix_size_regime='D+', norm_layer=nn.BatchNorm2d):
        super(ResNet_imagenet, self).__init__()
        self.norm_layer = norm_layer
        self.inplanes = inplanes
        self.conv1 = nn.Conv2d(3, inplanes, kernel_size=7, stride=2, padding=3, bias=False)
        self.bn1 = norm_layer(inplanes)
        self.relu = nn.ReLU(inplace=True)
        self.maxpool = nn.MaxPool2d(kernel_size=3, stride=2, padding=1)
        for i, (w, n, g) in enumerate(zip(width, layers, groups)):
            layer = self._make_layer(block=block, planes=w, blocks=n, expansion=expansion,
                                     stride=1 if i == 0 else 2, residual_block=residual_block, groups=g, mixup=mixup)
            if checkpoint_segments > 0:     # recompute in the backward pass (models/resnet.py:236-239)
                layer = CheckpointModule(layer, min(checkpoint_segments, n))
            setattr(self, 'layer%d' % (i + 1), layer)
        self.avgpool = nn.AdaptiveAvgPool2d(1)
        self.fc = nn.Linear(width[-1] * expansion, num_classes)
        init_model(self)

        steps_per_epoch = math.floor(self.num_train_images / (base_devices * base_device_batch))
        ramp_up_steps = steps_per_epoch * ramp_up_epochs

        def step_regime(milestones):
            first = {'epoch': milestones[0], 'optimizer': 'SGD', 'lr': scale_lr * 1e-1, 'momentum': 0.9,
                     'regularizer': weight_decay_config(1e-4)}
            return [first] + [{'epoch': e, 'lr': scale_lr * 10 ** -(k + 2)} for k, e in enumerate(milestones[1:])]

        self.regime = step_regime([0, 30, 60, 80])
        if 'cutmix' in regime:
            self.regime = step_regime([0, 75, 150, 225])
        if 'linear' in regime:
            # single phase with a per-step linear decay; with ramp_up_lr, a linear warm-up phase first.
            # (The reference's version of this branch raises a TypeError -- SURVEY appendix B -- this is the
            #  evident intent.)
            total = steps_per_epoch * epochs
            first = {'epoch': 0, 'optimizer': 'SGD', 'lr': scale_lr * 1e-1, 'momentum': 0.9,
                     'regularizer': weight_decay_config(1e-4),
                     'step_lambda': linear_scale(scale_lr * 1e-1, 0, total)}
            self.regime = [first]
            if ramp_up_lr:
                first['lr'] = 0
                first['step_lambda'] = linear_scale(0.1, scale_lr * 1e-1, ramp_up_steps)
                self.regime.append({'epoch': ramp_up_epochs,
                                    'step_lambda': linear_scale(scale_lr * 1e-1, 0,
                                                                steps_per_epoch * (epochs - ramp_up_epochs),
                                                                ramp_up_steps)})
                ramp_up_lr = False

        if 'sampled' in regime:  # Mix&Match: gradient smoothing + sampled input sizes
            self.regime[0]['regularizer'] = [{'name': 'GradSmooth', 'momentum': 0.9, 'log': False},
                                             weight_decay_config(1e-4)]
            ramp_up_lr = False
            self.data_regime = None

            def at(size):
                return mixsize_config(size, base_size=base_image_size, base_batch=base_device_batch,
                                      base_duplicates=base_duplicates, adapt_batch=mix_size_regime == 'B+',
                                      adapt_duplicates=mix_size_regime == 'D+')
            step = int(base_image_size / 7)
            if '144' in regime:
                plan = [(0.1, 1), (0.1, 0), (0.6, -3), (0.2, -4)]
            else:
                plan = [(0.8 / 6, -3), (0.8 / 6, -2), (0.8 / 6, -1), (0.2, 0), (0.8 / 6, 1), (0.8 / 6, 2), (0.8 / 6, 3)]
            self.sampled_data_regime = [(p, at(base_image_size + k * step)) for p, k in plan]
            self.data_eval_regime = [{'epoch': 0, 'input_size': base_image_size}]

        if ramp_up_lr and scale_lr > 1:  # large-batch linear LR warm-up
            self.regime[0]['step_lambda'] = linear_scale(0.1, 0.1 * scale_lr, ramp_up_steps)
            self.regime.insert(1, {'epoch': ramp_up_epochs, 'lr': scale_lr * 1e-1})


class ResNet_cifar(ResNet):
    def __init__(self, num_classes=10, inplanes=16, block=BasicBlock, depth=18, width=[16, 32, 64],
                 groups=[1, 1, 1], residual_block=None, regime='normal', dropout=None, mixup=False,
                 norm_layer=nn.BatchNorm2d):
        super(ResNet_cifar, self).__init__()
        self.norm_layer = norm_layer
        self.inplanes = inplanes
        n = int((depth - 2) / 6)
        self.conv1 = nn.Conv2d(3, inplanes, kernel_size=3, stride=1, padding=1, bias=False)
        self.bn1 = norm_layer(inplanes)
        self.relu = nn.ReLU(inplace=True)
        self.maxpool = nn.Identity()
        self.layer1 = self._make_layer(block, width[0], n, groups=groups[0], residual_block=residual_block,
                                       dropout=dropout, mixup=mixup)
        self.layer2 = self._make_layer(block, width[1], n, stride=2, groups=groups[1],
                                       residual_block=residual_block, dropout=dropout, mixup=mixup)
        self.layer3 = self._make_layer(block, width[2], n, stride=2, groups=groups[2],
                                       residual_block=residual_block, dropout=dropout, mixup=mixup)
        self.layer4 = nn.Identity()
        self.avgpool = nn.AdaptiveAvgPool2d(1)
        self.fc = nn.Linear(width[-1], num_classes)
        init_model(self)

        def step_regime(wd, lrs, epochs):
            first = {'epoch': 0, 'optimizer': 'SGD', 'lr': lrs[0], 'momentum': 0.9,
                     'regularizer': weight_decay_config(wd)}
            return [first] + [{'epoch': e, 'lr': lr} for e, lr in zip(epochs, lrs[1:])]

        self.regime = step_regime(1e-4, [1e-1, 1e-2, 1e-3, 1e-4], [81, 122, 164])
        if 'wide-resnet' in regime:
            self.regime = step_regime(5e-4, [1e-1, 2e-2, 4e-3, 8e-4], [60, 120, 160])
        if 'sampled' in regime:
            adapt_batch = 'B+' in regime
            adapt_duplicates = ('D+' in regime) or not adapt_batch

            def at(size):
                return mixsize_config(size, base_size=32, base_batch=64, base_duplicates=1,
                                      adapt_batch=adapt_batch, adapt_duplicates=adapt_duplicates)
            self.regime[0]['regularizer'] = [{'name': 'GradSmooth', 'momentum': 0.9, 'log': False},
                                             weight_decay_config(1e-4)]
            self.data_regime = None
            self.sampled_data_regime = [(0.3, at(32)), (0.2, at(48)), (0.3, at(24)), (0.2, at(16))]
            self.data_eval_regime = [{'epoch': 0, 'input_size': 32, 'scale_size': 32}]


_IMAGENET_DEPTHS = {
    18: dict(block=BasicBlock, layers=[2, 2, 2, 2], expansion=1),
    34: dict(block=BasicBlock, layers=[3, 4, 6, 3], expansion=1),
    50: dict(block=Bottleneck, layers=[3, 4, 6, 3]),
    101: dict(block=Bottleneck, layers=[3, 4, 23, 3]),
    152: dict(block=Bottleneck, layers=[3, 8, 36, 3]),
    200: dict(block=Bottleneck, layers=[3, 24, 36, 3]),
}


def _reject_out_of_scope(config):
    if config.pop('quantize', None):
        raise NotImplementedError("model-config 'quantize' selects a research variant outside the B200 hot path "
                                  "(SURVEY.md section 2, rows 24-25)")
    bn_norm = config.pop('bn_norm', None) or None
    if bn_norm not in _NORM_LAYERS:
        raise NotImplementedError("model-config bn_norm=%r is outside the B200 hot path (supported: 'L1'; "
                                  "SURVEY.md section 2, row 25)" % (bn_norm,))
    if bn_norm is not None:
        config['norm_layer'] = _NORM_LAYERS[bn_norm]


def resnet(**config):
    """Factory with the reference's config grammar: dataset in {imagenet*, cifar10, cifar100}, depth, and
    any constructor kwarg (regime, scale_lr, mix_size_regime, ...).  ``bn_norm='L1'`` builds every BatchNorm as
    models.modules.lp_norm.L1BatchNorm2d (the reference rebinds torch.nn.BatchNorm2d for the whole process instead;
    nothing global is touched here).  ``b200=True`` converts the model for the B200 kernel path (equivalent to
    calling engine.convert_b200 on the result)."""
    dataset = config.pop('dataset', 'imagenet')
    use_b200 = config.pop('b200', False)
    _reject_out_of_scope(config)
    if 'imagenet' in dataset:
        config.setdefault('num_classes', 1000)
        config.update(_IMAGENET_DEPTHS.get(config.pop('depth', 50), {}))
        model = ResNet_imagenet(**config)
    elif dataset in ('cifar10', 'cifar100') or 'cifar' in dataset:
        config.setdefault('num_classes', 100 if '100' in dataset else 10)
        config.setdefault('depth', 44)
        model = ResNet_cifar(block=BasicBlock, **config)
    else:
        raise ValueError('resnet: unknown dataset %r' % dataset)
    if use_b200:
        from ..engine import convert_b200
        model = convert_b200(model)
    return model


def resnet_se(**config):
    """ResNet with a squeeze-and-excitation gate on the residual branch of every block (models/resnet.py:434-436 of the
    reference): SURVEY.md section 8(f) row 4."""
    from .modules.se import SEBlock
    config['residual_block'] = SEBlock
    return resnet(**config)
