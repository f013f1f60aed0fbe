"""Command-line trainer with the reference's main.py flags (main.py:28-119 of eladhoffer/convNet.pytorch).

    python -m convnet.pytorch_b200.main --model resnet --model-config "{'depth': 20}" \
        --dataset synthetic_cifar10 --device cpu -b 64 --epochs 1                    # config C1 (plumbing)
    torchrun --nproc-per-node 8 -m convnet.pytorch_b200.main --model resnet --model-config "{'depth': 50}" \
        --dataset synthetic_imagenet --dtype bfloat16 -b 256                         # config C2 (B200 path)

Additions over the reference: ``--dtype bfloat16`` (compute type of the B200 kernels; parameters stay fp32
masters in the arena), ``synthetic_*`` datasets, ``--b200 {auto,on,off}`` (auto: on for CUDA devices),
``--device-augment`` (batch augmentation of the CIFAR transform done in the input relayout kernel, with the Resize of
the Mix&Match ``sampled*`` regimes),
``--device-resized-crop`` (the ImageNet RandomResizedCrop + flip resampled in the input relayout kernel),
``--device-scale-crop`` (the ImageNet evaluation Resize + CenterCrop resampled in the input relayout kernel),
``--device-decode`` (baseline JPEGs decoded on the GPU ahead of either device crop), and
rank/world are read from the torchrun environment when ``--local_rank`` is not given.
"""
import argparse
import json
import logging
import os
from ast import literal_eval
from datetime import datetime
from os import path, makedirs

import torch
import torch.distributed as dist
import torch.nn as nn

from . import models
from .data import DataRegime, SampledDataRegime
from .trainer import Trainer
from .utils.cross_entropy import CrossEntropyLoss
from .utils.log import setup_logging, ResultsLog, save_checkpoint, export_args_namespace
from .utils.misc import torch_dtypes, is_low_precision
from .utils.optim import OptimRegime
from .utils.param_filter import FilterModules, is_bn

model_names = sorted(name for name in models.__dict__
                     if name.islower() and not name.startswith('__') and callable(models.__dict__[name]))


def build_parser():
    p = argparse.ArgumentParser(description='ConvNet training on the B200 kernel path')
    a = p.add_argument
    a('--config-file', default=None, help='json configuration file')
    a('--results-dir', metavar='RESULTS_DIR', default='./results', help='results dir')
    a('--save', metavar='SAVE', default='', help='saved folder')
    a('--datasets-dir', metavar='DATASETS_DIR', default='~/Datasets', help='datasets dir')
    a('--dataset', metavar='DATASET', default='imagenet', help='dataset name or folder')
    a('--model', '-a', metavar='MODEL', default='resnet', choices=model_names,
      help='model architecture: ' + ' | '.join(model_names))
    a('--input-size', type=int, default=None, help='image input size')
    a('--model-config', default='', help='additional architecture configuration')
    a('--dtype', default='float', help='type of tensor: ' + ' | '.join(torch_dtypes.keys()))
    a('--device', default='cuda', help='device assignment ("cpu" or "cuda")')
    a('--device-ids', default=[0], type=int, nargs='+', help='device ids assignment (e.g 0 1 2 3)')
    a('--world-size', default=-1, type=int, help='number of distributed processes')
    a('--local_rank', '--local-rank', default=-1, type=int, help='rank of distributed processes')
    a('--dist-init', default='env://', type=str, help='init used to set up distributed training')
    a('--dist-backend', default='nccl', type=str, help='distributed backend')
    a('-j', '--workers', default=8, type=int, metavar='N', help='number of data loading workers')
    a('--epochs', default=90, type=int, metavar='N', help='number of total epochs to run')
    a('--start-epoch', default=-1, type=int, metavar='N', help='manual epoch number (-1: from checkpoint or 0)')
    a('-b', '--batch-size', default=256, type=int, metavar='N', help='mini-batch size PER PROCESS')
    a('--eval-batch-size', default=-1, type=int, help='mini-batch size for evaluation (default: same)')
    a('--optimizer', default='SGD', type=str, metavar='OPT', help='optimizer function used')
    a('--drop-optim-state', action='store_true', default=False, help='do not save optimizer state for resume')
    a('--save-all', action='store_true', default=False, help='save checkpoint for every epoch')
    a('--label-smoothing', default=0, type=float, help='label smoothing coefficient')
    a('--sync-bn', action='store_true', default=False, help='synchronize batch-norm statistics across ranks')
    a('--mixup', default=None, type=float, help='mixup alpha coefficient - default None')
    a('--cutmix', default=None, type=float,
      help='cutmix alpha coefficient - default None (with --mixup as well: CutMix with the --mixup alpha)')
    a('--duplicates', default=1, type=int, help='number of augmentations over single example')
    a('--chunk-batch', default=1, type=int, help='chunk batch size for multiple passes (training)')
    a('--cutout', action='store_true', default=False,
      help='cutout augmentations (ignored for synthetic data unless --device-augment)')
    a('--device-augment', action='store_true', default=False,
      help='CIFAR training: ship uint8 images and per-copy draws, and crop / resize (Mix&Match size regimes) / flip / '
           'cutout the --duplicates copies inside the input relayout on the GPU')
    a('--device-resized-crop', action='store_true', default=False,
      help='ImageNet training: the loader workers only decode and draw the crop boxes and flips; the input relayout '
           'on the GPU resamples the crops (Pillow-exact bilinear), flips and normalises them')
    a('--device-scale-crop', action='store_true', default=False,
      help='ImageNet validation: the loader workers only decode; the input relayout on the GPU resizes (Pillow-exact '
           'bilinear), centre-crops and normalises the images')
    a('--device-decode', action='store_true', default=False,
      help='ImageNet, with --device-resized-crop (training) and / or --device-scale-crop (validation): the loader '
           'workers only read the files and parse their headers; baseline JPEGs are decoded on the GPU into the '
           'regions the crops read, byte for byte what Pillow decodes (other files are decoded by the workers)')
    a('--autoaugment', action='store_true', default=False, help='autoaugment policies (ignored for synthetic data)')
    a('--grad-clip', default=-1, type=float, help='maximum grad norm value, -1 for none')
    a('--loss-scale', default=1, type=float, help='loss scale for mixed precision training')
    a('--lr', '--learning-rate', default=0.1, type=float, metavar='LR', help='initial learning rate')
    a('--momentum', default=0.9, type=float, metavar='M', help='momentum')
    a('--weight-decay', '--wd', default=0, type=float, metavar='W', help='weight decay')
    a('--print-freq', '-p', default=10, type=int, metavar='N', help='print frequency')
    a('--adapt-grad-norm', default=None, type=int, help='adapt gradient scale frequency')
    a('--resume', default='', type=str, metavar='PATH', help='path to latest checkpoint')
    a('-e', '--evaluate', type=str, metavar='FILE', help='evaluate model FILE on validation set')
    a('--seed', default=123, type=int, help='random seed')
    a('--b200', default='auto', choices=['auto', 'on', 'off'], help='use the B200 kernel path (auto: on CUDA)')
    a('--max-steps', default=None, type=int, help='stop each training epoch after N steps (smoke runs)')
    return p


parser = build_parser()


def main(argv=None):
    args = parser.parse_args(argv)
    if args.config_file is not None:
        with open(args.config_file) as f:
            parser.set_defaults(**json.loads(f.read()))
        args = parser.parse_args(argv)
    return main_worker(args)


def _model_dataset_name(dataset):
    """The factories dispatch on 'imagenet' in name / == 'cifar10': map synthetic names onto those."""
    return dataset.replace('synthetic_', '')


def main_worker(args):
    best_prec1 = 0
    dtype = torch_dtypes.get(args.dtype)
    if dtype is None:
        raise ValueError('unknown --dtype %r' % args.dtype)
    torch.manual_seed(args.seed)
    if args.evaluate:
        args.results_dir = '/tmp'
    if args.save == '':
        args.save = datetime.now().strftime('%Y-%m-%d_%H-%M-%S')
    save_path = path.join(args.results_dir, args.save)

    env_world = int(os.environ.get('WORLD_SIZE', '1'))
    if args.local_rank < 0 and env_world > 1:  # launched by torchrun
        args.local_rank = int(os.environ.get('LOCAL_RANK', '0'))
        args.world_size = env_world
    args.distributed = args.local_rank >= 0 or args.world_size > 1
    if args.distributed:
        if 'cuda' not in args.device and args.dist_backend == 'nccl':
            args.dist_backend = 'gloo'
        if args.dist_init == 'env://' and 'RANK' in os.environ:
            dist.init_process_group(backend=args.dist_backend, init_method=args.dist_init)
        else:
            dist.init_process_group(backend=args.dist_backend, init_method=args.dist_init,
                                    world_size=args.world_size, rank=args.local_rank)
        args.world_size = dist.get_world_size()
        rank = dist.get_rank()
        args.device_ids = [args.local_rank if 'LOCAL_RANK' not in os.environ else int(os.environ['LOCAL_RANK'])]
    else:
        rank = 0
    is_main = rank == 0

    if is_main:
        makedirs(save_path, exist_ok=True)
        export_args_namespace(args, path.join(save_path, 'config.json'))
    setup_logging(path.join(save_path, 'log.txt'), resume=args.resume != '', dummy=not is_main)
    results = ResultsLog(path.join(save_path, 'results'), title='Training Results - %s' % args.save) \
        if is_main else None
    logging.info('saving to %s', save_path)
    logging.debug('run arguments: %s', args)

    on_cuda = 'cuda' in args.device and torch.cuda.is_available()
    if on_cuda:
        torch.cuda.manual_seed_all(args.seed)
        torch.cuda.set_device(args.device_ids[0])
        args.device = 'cuda:%d' % args.device_ids[0]
    else:
        args.device_ids = None
    if args.device_decode and not (args.device_resized_crop or args.device_scale_crop):
        raise NotImplementedError('--device-decode decodes into the regions of --device-resized-crop or '
                                  '--device-scale-crop; set one of them')
    if args.device_decode and not on_cuda:
        raise NotImplementedError('--device-decode decodes on the GPU: it needs a CUDA device')
    use_b200 = args.b200 == 'on' or (args.b200 == 'auto' and on_cuda)
    if use_b200 and not on_cuda:
        raise RuntimeError('--b200 on requires a CUDA device: the B200 kernel path has no CPU fallback')

    # ---- model ----
    logging.info('creating model %s', args.model)
    model_config = {'dataset': _model_dataset_name(args.dataset)}
    if args.model_config != '':
        model_config = dict(model_config, **literal_eval(args.model_config))
    model = models.__dict__[args.model](**model_config)
    if args.sync_bn:
        from .models.modules.lp_norm import L1BatchNorm2d
        if any(isinstance(m, L1BatchNorm2d) for m in model.modules()):
            raise NotImplementedError('--sync-bn is not implemented for L1 BatchNorm (bn_norm=\'L1\')')
        from .models.modules.checkpoint import CheckpointModule
        if any(isinstance(m, CheckpointModule) for m in model.modules()):
            raise NotImplementedError('--sync-bn is not implemented with checkpoint_segments')
    if args.sync_bn and not use_b200:
        model = nn.SyncBatchNorm.convert_sync_batchnorm(model)
    logging.info('created model with configuration: %s', model_config)
    logging.info('number of parameters: %d', sum(p.nelement() for p in model.parameters()))

    optim_state_dict = None
    checkpoint_file = args.evaluate or None
    if args.resume:
        checkpoint_file = args.resume
        if path.isdir(checkpoint_file):
            if results is not None and path.isfile(path.join(checkpoint_file, 'results.csv')):
                results.load(path.join(checkpoint_file, 'results.csv'))
            checkpoint_file = path.join(checkpoint_file, 'model_best.pth.tar')
    if checkpoint_file:
        if not path.isfile(checkpoint_file):
            parser.error('invalid checkpoint: {}'.format(checkpoint_file))
        checkpoint = torch.load(checkpoint_file, map_location='cpu', weights_only=False)
        model.load_state_dict(checkpoint['state_dict'])
        if args.resume:
            if args.start_epoch < 0:
                args.start_epoch = checkpoint['epoch']
            best_prec1 = checkpoint.get('best_prec1', 0)
            optim_state_dict = checkpoint.get('optim_state_dict', None)
        logging.info("loaded checkpoint '%s' (epoch %s)", checkpoint_file, checkpoint.get('epoch'))

    # ---- loss, precision, device placement ----
    loss_params = {}
    if args.label_smoothing > 0:
        loss_params['smooth_eps'] = args.label_smoothing
    criterion = getattr(model, 'criterion', CrossEntropyLoss)(**loss_params)
    if use_b200:
        from .engine import convert_b200
        model = convert_b200(model, args.device)   # fp32 masters in the arena, bf16 compute inside the kernels
        if args.sync_bn and args.distributed:
            from .engine import enable_sync_batchnorm
            enable_sync_batchnorm(model)             # statistics all-reduced between the conv epilogue and bn_finalize
        criterion.to(args.device)
    else:
        criterion.to(args.device, dtype)
        model.to(args.device, dtype)
        if is_low_precision(args.dtype):  # batch-norm always in float (main.py:239-240 of the reference)
            FilterModules(model, module=is_bn).to(dtype=torch.float)

    # ---- optimizer regime ----
    optim_regime = getattr(model, 'regime', [{'epoch': 0, 'optimizer': args.optimizer, 'lr': args.lr,
                                              'momentum': args.momentum, 'weight_decay': args.weight_decay}])
    optimizer = optim_regime if isinstance(optim_regime, OptimRegime) else \
        OptimRegime(model, optim_regime, use_float_copy=(not use_b200) and is_low_precision(args.dtype))
    if optim_state_dict is not None:
        optimizer.update(max(args.start_epoch, 0), 0)   # instantiate the optimizer class of the phase first
        optimizer.load_state_dict(optim_state_dict)

    trainer = Trainer(model, criterion, optimizer, device_ids=args.device_ids, device=args.device, dtype=dtype,
                      print_freq=args.print_freq, distributed=args.distributed, local_rank=args.local_rank,
                      mixup=args.mixup, cutmix=args.cutmix, loss_scale=args.loss_scale, grad_clip=args.grad_clip,
                      adapt_grad_norm=args.adapt_grad_norm)

    # ---- data ----
    args.eval_batch_size = args.eval_batch_size if args.eval_batch_size > 0 else args.batch_size
    val_data = DataRegime(getattr(model, 'data_eval_regime', None),
                          defaults={'datasets_path': args.datasets_dir, 'name': args.dataset, 'split': 'val',
                                    'augment': False, 'input_size': args.input_size,
                                    'batch_size': args.eval_batch_size, 'shuffle': False,
                                    'num_workers': args.workers, 'pin_memory': True, 'drop_last': False,
                                    'device_scale_crop': args.device_scale_crop,
                                    'device_decode': args.device_decode and args.device_scale_crop})
    if args.evaluate:
        res = trainer.validate(val_data.get_loader())
        logging.info(res)
        return res

    train_defaults = {'datasets_path': args.datasets_dir, 'name': args.dataset, 'split': 'train', 'augment': True,
                      'input_size': args.input_size, 'batch_size': args.batch_size, 'shuffle': True,
                      'num_workers': args.workers, 'pin_memory': True, 'drop_last': True,
                      'distributed': args.distributed, 'duplicates': args.duplicates,
                      'autoaugment': args.autoaugment, 'cutout': {'holes': 1, 'length': 16} if args.cutout else None,
                      'device_augment': args.device_augment, 'device_resized_crop': args.device_resized_crop,
                      'device_decode': args.device_decode and args.device_resized_crop}
    if hasattr(model, 'sampled_data_regime'):
        probs, configs = zip(*model.sampled_data_regime)
        train_data = SampledDataRegime([DataRegime(None, defaults={**train_defaults, **cfg}) for cfg in configs],
                                       probs)
    else:
        train_data = DataRegime(getattr(model, 'data_regime', None), defaults=train_defaults)

    logging.info('optimization regime: %s', optim_regime)
    logging.info('data regime: %s', train_data)
    args.start_epoch = max(args.start_epoch, 0)
    trainer.training_steps = args.start_epoch * len(train_data)
    last = {}
    for epoch in range(args.start_epoch, args.epochs):
        trainer.epoch = epoch
        train_data.set_epoch(epoch)
        val_data.set_epoch(epoch)
        logging.info('\nStarting Epoch: {0}\n'.format(epoch + 1))
        loader = train_data.get_loader()
        if args.max_steps is not None:
            trainer.model.train()
            train_results = trainer.forward(loader, num_steps=args.max_steps - 1, training=True,
                                            chunk_batch=args.chunk_batch)
            trainer.model.eval()
            with torch.no_grad():
                val_results = trainer.forward(val_data.get_loader(), num_steps=args.max_steps - 1, training=False)
        else:
            train_results = trainer.train(loader, chunk_batch=args.chunk_batch)
            val_results = trainer.validate(val_data.get_loader())
        last = {'train': train_results, 'val': val_results}
        if not is_main:
            continue
        is_best = val_results['prec1'] > best_prec1
        best_prec1 = max(val_results['prec1'], best_prec1)
        save_checkpoint({'epoch': epoch + 1, 'model': args.model, 'config': args.model_config,
                         'state_dict': model.state_dict(),
                         'optim_state_dict': None if args.drop_optim_state else optimizer.state_dict(),
                         'best_prec1': best_prec1}, is_best, path=save_path, save_all=args.save_all)
        logging.info('\nResults - Epoch: {0}\n'
                     'Training Loss {train[loss]:.4f} \tTraining Prec@1 {train[prec1]:.3f} \t'
                     'Training Prec@5 {train[prec5]:.3f} \tValidation Loss {val[loss]:.4f} \t'
                     'Validation Prec@1 {val[prec1]:.3f} \tValidation Prec@5 {val[prec5]:.3f} \t\n'
                     .format(epoch + 1, train=train_results, val=val_results))
        values = dict(epoch=epoch + 1, steps=trainer.training_steps)
        values.update({'training ' + k: v for k, v in train_results.items()})
        values.update({'validation ' + k: v for k, v in val_results.items()})
        results.add(**values)
        results.save()
    if args.distributed:
        trainer.release_graphs()       # captured steps hold NCCL work: drop them before the process group goes away
        dist.barrier()
    return last


if __name__ == '__main__':
    main()
