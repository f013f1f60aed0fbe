"""MobileNet (v1) on the reference's factory contract (models/mobilenet.py:39-178): a 3x3/s2 stem followed by 13
depthwise-separable units -- depthwise 3x3 (WITH bias, as in the reference, whose nn.Conv2d call leaves the default
bias=True) -> BN -> ReLU -> 1x1 -> BN -> ReLU -- global average pooling and a linear classifier.  Module names
(``features.{i}``, ``features.{i}.components.{j}``, ``fc``) match the reference so checkpoints interchange; weight decay
skips the depthwise convolutions (models/mobilenet.py:23-36).  SURVEY.md section 8(f) row 4: a neighbour family that runs
on the same kernels as MobileNet-v2 (depthwise CUDA-core kernels + wgmma 1x1 convolutions)."""
import torch.nn as nn

__all__ = ['mobilenet']


def nearby_int(n):
    return int(round(n))


def weight_decay_config(value=1e-4, log=True):
    def decayed(m):
        dense_conv = isinstance(m, nn.Conv2d) and m.groups != m.in_channels
        return dense_conv or isinstance(m, nn.Linear)
    return {'name': 'WeightDecay', 'value': value, 'log': log,
            'filter': {'parameter_name': lambda n: not n.endswith('bias'), 'module': decayed}}


class DepthwiseSeparableFusedConv2d(nn.Module):
    def __init__(self, in_channels, out_channels, kernel_size, stride=1, padding=0):
        super(DepthwiseSeparableFusedConv2d, self).__init__()
        self.components = nn.Sequential(
            nn.Conv2d(in_channels, in_channels, kernel_size, stride=stride, padding=padding, groups=in_channels),
            nn.BatchNorm2d(in_channels), nn.ReLU(inplace=True),
            nn.Conv2d(in_channels, out_channels, 1, bias=False), nn.BatchNorm2d(out_channels), nn.ReLU(inplace=True))

    def forward(self, x):
        return self.components(x)


class MobileNet(nn.Module):
    _b200 = None

    def __init__(self, width=1., shallow=False, regime=None, num_classes=1000):
        super(MobileNet, self).__init__()
        num_classes = num_classes or 1000
        width = width or 1.
        w = lambda c: nearby_int(width * c)  # noqa: E731
        plan = [(32, 64, 1), (64, 128, 2), (128, 128, 1), (128, 256, 2), (256, 256, 1), (256, 512, 2)]
        if not shallow:
            plan += [(512, 512, 1)] * 5
        plan += [(512, 1024, 2), (1024, 1024, 1)]      # the reference keeps stride 1 in the last unit
        layers = [nn.Conv2d(3, w(32), kernel_size=3, stride=2, padding=1, bias=False), nn.BatchNorm2d(w(32)),
                  nn.ReLU(inplace=True)]
        layers += [DepthwiseSeparableFusedConv2d(w(a), w(b), kernel_size=3, stride=s, padding=1) for a, b, s in plan]
        self.features = nn.Sequential(*layers)
        self.avg_pool = nn.AdaptiveAvgPool2d(1)
        self.fc = nn.Linear(w(1024), num_classes)
        # the reference defines an init_model() in this file but never calls it: torch's default initialisation stays
        steps = [(0, 1e-1), (30, 1e-2), (60, 1e-3), (80, 1e-4)]
        scale = 4 if regime == 'small' else 1
        self.regime = [{'epoch': 0, 'optimizer': 'SGD', 'momentum': 0.9, 'lr': scale * steps[0][1],
                        'regularizer': weight_decay_config(1e-4)}] + \
                      [{'epoch': e, 'lr': scale * lr} for e, lr in steps[1:]]
        if regime == 'small':
            self.data_regime = [{'epoch': 0, 'input_size': 128, 'batch_size': 512},
                                {'epoch': 80, 'input_size': 224, 'batch_size': 128}]
            self.data_eval_regime = [{'epoch': 0, 'input_size': 128, 'batch_size': 1024},
                                     {'epoch': 80, 'input_size': 224, 'batch_size': 512}]

    def forward(self, x):
        if self._b200 is not None:
            return self._b200.forward(x)
        x = self.avg_pool(self.features(x))
        return self.fc(x.view(x.size(0), -1))


def mobilenet(**config):
    """MobileNet-v1 ("MobileNets: Efficient Convolutional Neural Networks for Mobile Vision Applications")."""
    dataset = config.pop('dataset', 'imagenet')
    use_b200 = config.pop('b200', False)
    assert 'imagenet' in dataset, 'mobilenet is defined for ImageNet-shaped inputs'
    model = MobileNet(**config)
    if use_b200:
        from ..engine import convert_b200
        model = convert_b200(model)
    return model
