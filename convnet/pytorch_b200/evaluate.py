"""Checkpoint evaluation CLI with the reference's evaluate.py flags (evaluate.py:28-193 of eladhoffer/convNet.pytorch).

    python -m convnet.pytorch_b200.evaluate results/run/checkpoint.pth.tar --dataset synthetic_imagenet \
        [--calibrate-bn] [--absorb-bn] [--avg-out --duplicates 4] [-b 256] [--device cuda] [--device-scale-crop]

Flow (evaluate.py:101-193): load the checkpoint (its ``model`` / ``config`` entries override the command line) ->
build the model from the registry -> ``load_state_dict`` -> optional ``--absorb-bn`` -> criterion -> Trainer ->
optional ``--calibrate-bn`` (200 training-mode forward passes with cumulative-average BN statistics,
trainer.py:277-285) -> ``Trainer.validate(loader, average_output=--avg-out)``.

On the B200 path ``--absorb-bn`` selects the kernels with BatchNorm folded into the convolution -- the recipe of the
reference's utils/absorb_bn.py:18-48 (w' = w * gamma / sqrt(var + eps), b' = beta - mean * gamma / sqrt(var + eps))
applied to the bf16 kernel weights and the epilogue bias, so every conv + BN + (residual) + ReLU unit is ONE launch;
without the flag the convolution and the BatchNorm-apply kernels run separately, as the reference's modules do.  The
checkpoint's state_dict is never mutated (the reference rewrites conv weights in place); with ``--calibrate-bn`` the
statistics are re-estimated first and folded afterwards, which evaluates the same function as the reference's
"absorb, reset statistics, calibrate" order.  On CPU / non-converted models the flag folds the torch modules exactly
like ``search_absorb_bn``.
"""
import argparse
import logging
import os
from ast import literal_eval
from datetime import datetime

import torch
import torch.nn as nn

from . import models
from .data import DataRegime
from .main import model_names, _model_dataset_name
from .trainer import Trainer
from .utils.cross_entropy import CrossEntropyLoss
from .utils.log import setup_logging
from .utils.misc import torch_dtypes


def build_parser():
    p = argparse.ArgumentParser(description='ConvNet evaluation on the B200 kernel path')
    a = p.add_argument
    a('evaluate', type=str, help='evaluate model FILE on validation set')
    a('--results-dir', metavar='RESULTS_DIR', default='./results', help='results dir')
    a('--save', metavar='SAVE', default='', help='saved folder')
    a('--datasets-dir', metavar='DATASETS_DIR', default='~/Datasets', help='datasets dir')
    a('--dataset', metavar='DATASET', default='imagenet', help='dataset name or folder')
    a('--model', '-a', metavar='MODEL', default='resnet', choices=model_names, help='model architecture')
    a('--input-size', type=int, default=None, help='image input size')
    a('--model-config', default='', help='additional architecture configuration')
    a('--dtype', default='float', help='type of tensor: ' + ' | '.join(torch_dtypes.keys()))
    a('--device', default='cuda', help='device assignment ("cpu" or "cuda")')
    a('--device-ids', default=[0], type=int, nargs='+', help='device ids assignment')
    a('-j', '--workers', default=8, type=int, metavar='N', help='number of data loading workers')
    a('-b', '--batch-size', default=256, type=int, metavar='N', help='mini-batch size')
    a('--label-smoothing', default=0, type=float, help='label smoothing coefficient')
    a('--mixup', default=None, type=float, help='mixup alpha coefficient - accepted for CLI parity, unused in evaluation')
    a('--duplicates', default=1, type=int, help='number of augmentations over single example')
    a('--augment', action='store_true', default=False, help='perform augmentations')
    a('--device-scale-crop', action='store_true', default=False,
      help='ImageNet: the loader workers only decode; the input relayout on the GPU resizes (Pillow-exact bilinear), '
           'centre-crops and normalises the images')
    a('--calibrate-bn', action='store_true', default=False, help='calibrate bn stats')
    a('--calibrate-steps', default=200, type=int, help='forward passes of --calibrate-bn (reference: 200)')
    a('--avg-out', action='store_true', default=False, help='average outputs over the duplicates')
    a('--absorb-bn', action='store_true', default=False, help='absorb batch-norm before evaluation')
    a('--print-freq', '-p', default=10, type=int, metavar='N', help='print frequency')
    a('--seed', default=123, type=int, help='random seed')
    a('--b200', default='auto', choices=['auto', 'on', 'off'], help='use the B200 kernel path (auto: on CUDA)')
    return p


parser = build_parser()


def absorb_bn_torch(model):
    """utils/absorb_bn.py:52-66 for plain torch modules: fold every BatchNorm that directly follows a Conv2d / Linear
    sibling into it and replace the BatchNorm by Identity.  An L1 BatchNorm folds with its running scale
    (running_var holds s: y = (x - running_mean) * running_var * weight + bias)."""
    from .models.modules.lp_norm import L1BatchNorm2d
    prev = None
    for name, m in list(model.named_children()):
        if isinstance(m, (nn.BatchNorm2d, nn.BatchNorm1d, L1BatchNorm2d)) and isinstance(prev, (nn.Conv2d, nn.Linear)):
            with torch.no_grad():
                if isinstance(m, L1BatchNorm2d):
                    inv = m.running_var * m.weight
                else:
                    inv = (m.running_var + m.eps).rsqrt() * (m.weight if m.affine else 1.0)
                shape = (-1,) + (1,) * (prev.weight.dim() - 1)
                prev.weight.mul_(inv.view(shape))
                bias = prev.bias if prev.bias is not None else torch.zeros_like(m.running_mean)
                bias = (bias - m.running_mean) * inv + (m.bias if m.affine else 0.0)
                prev.bias = nn.Parameter(bias)
            setattr(model, name, nn.Identity())
            m = getattr(model, name)
        else:
            absorb_bn_torch(m)
        prev = m
    return model


def main(argv=None):
    return main_worker(parser.parse_args(argv))


def main_worker(args):
    dtype = torch_dtypes.get(args.dtype)
    torch.manual_seed(args.seed)
    if args.save == '':
        args.save = datetime.now().strftime('%Y-%m-%d_%H-%M-%S')
    save_path = os.path.join('/tmp' if args.evaluate else args.results_dir, args.save)
    os.makedirs(save_path, exist_ok=True)
    setup_logging(os.path.join(save_path, 'log.txt'))
    cuda = 'cuda' in args.device and torch.cuda.is_available()
    if cuda:
        torch.cuda.manual_seed_all(args.seed)
        torch.cuda.set_device(args.device_ids[0])
    else:
        args.device_ids = None
    if not os.path.isfile(args.evaluate):
        parser.error('invalid checkpoint: {}'.format(args.evaluate))
    checkpoint = torch.load(args.evaluate, map_location='cpu', weights_only=False)
    args.model = checkpoint.get('model', args.model)            # checkpoint info overrides the command line
    args.model_config = checkpoint.get('config', args.model_config)
    model_config = {'dataset': _model_dataset_name(args.dataset)}
    if args.model_config != '':
        cfg = args.model_config if isinstance(args.model_config, dict) else literal_eval(args.model_config)
        model_config = dict(model_config, **cfg)
    model_config.pop('b200', None)
    model = models.__dict__[args.model](**model_config)
    logging.info('created model with configuration: %s', model_config)
    logging.info('number of parameters: %d', sum(p.nelement() for p in model.parameters()))
    model.load_state_dict(checkpoint['state_dict'])
    logging.info("loaded checkpoint '%s' (epoch %s)", args.evaluate, checkpoint.get('epoch'))

    use_b200 = args.b200 == 'on' or (args.b200 == 'auto' and cuda)
    if use_b200:
        from . import engine
        engine.convert_b200(model, torch.device('cuda', args.device_ids[0]))
        engine.FOLD_BN_EVAL = bool(args.absorb_bn)     # folded conv+BN kernels <=> utils/absorb_bn.py semantics
        dtype = torch.float
    else:
        if args.absorb_bn and not args.calibrate_bn:
            absorb_bn_torch(model)
        model.to(args.device, dtype)

    loss_params = {'smooth_eps': args.label_smoothing} if args.label_smoothing > 0 else {}
    criterion = getattr(model, 'criterion', CrossEntropyLoss)(**loss_params)
    criterion.to(args.device)
    trainer = Trainer(model, criterion, device_ids=args.device_ids, device=args.device, dtype=dtype,
                      mixup=args.mixup, print_freq=args.print_freq)
    common = {'datasets_path': args.datasets_dir, 'name': args.dataset, 'input_size': args.input_size,
              'batch_size': args.batch_size, 'num_workers': args.workers, 'pin_memory': cuda, 'drop_last': False}
    val_data = DataRegime(None, defaults=dict(common, split='val', augment=args.augment, shuffle=False,
                                              duplicates=args.duplicates, device_scale_crop=args.device_scale_crop))
    if args.calibrate_bn:
        train_data = DataRegime(None, defaults=dict(common, split='train', augment=True, shuffle=True))
        trainer.calibrate_bn(train_data.get_loader(), num_steps=args.calibrate_steps)
        if use_b200:
            model._b200.arena.version += 1            # running statistics moved: folded weights are stale
        elif args.absorb_bn:
            absorb_bn_torch(model)
    results = trainer.validate(val_data.get_loader(), average_output=args.avg_out)
    logging.info(results)
    print(results)
    return results


if __name__ == '__main__':
    main()
