"""Census of the convolutions the engine really launches, replayed exactly against fp64.

For each configuration of CONFIGS (models built by their own factories; the Mix&Match sizes and row counts read from
``model.sampled_data_regime``) the library calls of one ``Runtime.train_step`` and of two eval forwards (BatchNorm
folded into the convolutions, and not folded) are recorded by wrapping every public function of
``convnet.pytorch_b200.ops``, which the engine calls as ``ops.X`` throughout.  Every conv_fprop / conv_dgrad /
conv_wgrad call becomes a case of tests/test_gpu_conv_sweep.py -- its descriptor, epilogue (bias, residual, activation,
fp32 output, fused statistics) and direction, at the real batch -- and grouped operands are recognised by their pointer:
fprop / dgrad weights as the output of an earlier group_weight_pack, weight gradients by the group_wgrad_unpack that
reads them.  A call that does not map onto a case fails the test, and so does an ops entry point missing from
ELSEWHERE, the table of where every other kernel is verified.

The unique cases run the sweep's tier 1 (sparse integer operands, bit for bit against the fp64 reference rounded once)
for every configuration and its tier 2 (normal bf16 operands, rounding bounds) for the CIFAR configurations and at
224 px.  The BatchNorm shapes whose channel count is outside the kernel sweep's list run that sweep's tier-1
bn_stats / bn_apply / bn_backward checks.  test_census_witnesses_and_report fails when a shape the census exists for is
no longer recorded and exact, and prints the census.

The whole file (16 configurations, 1556 unique convolutions) takes 50 s on an NVIDIA H100 80GB HBM3 at a 700 W power
limit; operands are drawn on the device.

CIFAR resnet_se (depth 20) is not in the table: its 16-channel SE gate has a hidden width of 1, which the engine
refuses.
"""
import inspect
import math
import time

import pytest
import torch

import test_gpu_conv_sweep as cs_sweep
import test_gpu_kernel_sweep as k_sweep

pytestmark = pytest.mark.gpu

CONV = ('conv_fprop', 'conv_dgrad', 'conv_wgrad')
DIRS = {'conv_fprop': 'f', 'conv_dgrad': 'd', 'conv_wgrad': 'w'}
DESC_FIELDS = ('N', 'H', 'W', 'C', 'K', 'R', 'S', 'stride', 'pad_h', 'pad_w', 'P', 'Q', 'x_pixel_stride',
               'x_row_stride', 'x_image_stride', 'window')

# every other ops entry point the engine may call -> where it is verified at the shapes the engine gives it
_KS, _OPS = 'test_gpu_kernel_sweep.py', 'test_gpu_ops.py'
ELSEWHERE = {
    'bn_stats': _KS + ' (+ this census at channel counts outside its list)',
    'bn_apply': _KS + ' (+ this census at channel counts outside its list)',
    'bn_bwd_reduce': _KS + ' (+ this census at channel counts outside its list)',
    'bn_bwd_dx': _KS + ' (+ this census at channel counts outside its list)',
    'bn_finalize': _KS + '::test_bn_finalize; the sums it reads are the fused statistics replayed here',
    'bn_eval_coeffs': _KS + '::test_bn_eval_coeffs',
    'bn_apply_maxpool': _KS + '::test_bn_apply_maxpool',
    'maxpool_fwd': _KS + '::test_maxpool',
    'maxpool_bwd': _KS + '::test_maxpool',
    'avgpool_fwd': _KS + '::test_avgpool',
    'avgpool_bwd': _KS + '::test_avgpool',
    'dwconv_fprop': _KS + '::test_depthwise',
    'dwconv_dgrad': _KS + '::test_depthwise',
    'dwconv_wgrad': _KS + '::test_depthwise',
    'se_pool': _KS + '::test_se',
    'se_scale_fwd': _KS + '::test_se',
    'se_bwd_reduce': _KS + '::test_se',
    'se_bwd_dx': _KS + '::test_se',
    'act_bwd': _KS + '::test_act_bwd',
    'softmax_ce': _KS + '::test_softmax_ce',
    'colsum_bf16': _KS + '::test_colsum',
    'bn_l1_stats': 'test_gpu_l1_norm.py',
    'bn_l1_eval_coeffs': 'test_gpu_l1_norm.py',
    'bn_l1_bwd_dx': 'test_gpu_l1_norm.py',
    'bn_apply_dropout': 'test_gpu_dropout.py',
    'bn_bwd_reduce_dropout': 'test_gpu_dropout.py',
    'bn_bwd_dx_dropout': 'test_gpu_dropout.py',
    'dropout_threshold': 'test_dropout_cpu.py (host-side keep threshold and scale)',
    'input_prep': _OPS + ', test_gpu_mixup.py',
    'cast_bf16': _OPS,
    'weight_transpose': _OPS,
    'weight_transpose_batched': _OPS,
    'transpose_jobs': _OPS + ' (host-side job table of weight_transpose_batched)',
    'stem_weight_to_s2d': 'test_gpu_conv_sweep.py::test_stem_weight_relayout',
    'stem_wgrad_from_s2d': 'test_gpu_conv_sweep.py::test_stem_weight_relayout',
    'make_desc': 'host-side descriptor; every descriptor it made for a convolution is replayed here',
    'out_size': 'host-side arithmetic of make_desc',
    'can_fuse_bn_stats': 'host-side rule; the statistics epilogues it selects are replayed here',
    'bn_workspace_floats': 'host-side size query',
    'bn_act_mask_bytes': 'host-side size arithmetic; the masks are checked by ' + _KS,
}
BN_FAMILY = ('bn_stats', 'bn_apply', 'bn_bwd_reduce', 'bn_bwd_dx')

# tier-2 bounds of the census: c for bf16 and fp32 outputs, rel-L2 limits for bf16 and fp32 outputs.  The sweep's are
# calibrated on short reductions; the engine's weight gradients reduce up to 32768 products per element (WRN-28-10 at
# batch 128), in long fp32 chains.  Measured on an NVIDIA H100 80GB HBM3 (700 W power limit): worst excess ratio
# 5.0e-7 for bf16 outputs (WRN-28-10's 640-channel 3x3 fprop; 1.9x below 2^-20), 1.02e-6 for fp32 outputs (the 640-channel 3x3 weight gradient at 8 x 8
# px; 3.7x below 2^-18, above the sweep's 2^-20); fp32 rel-L2 2.02e-5 (the 320-channel one at 16 x 16 px).
COEF = (2.0 ** -20, 2.0 ** -18, 4e-3, 8e-5)


# ------------------------------------------------------------------------------------------------ the table
def _models():
    from convnet.pytorch_b200 import models
    return models


def _sampled(model):
    return sorted({(r['input_size'], r['batch_size'] * r['duplicates']) for _, r in model.sampled_data_regime})


def _cifar(factory, batch, **kw):
    return dict(make=lambda: getattr(_models(), factory)(dataset='cifar10', **kw),
                sizes=lambda m: [(32, batch)], rounding=None)


def _imagenet(factory, batch, rounding=(224,), **kw):
    return dict(make=lambda: getattr(_models(), factory)(dataset='imagenet', **kw),
                sizes=lambda m: [(224, batch)], rounding=rounding)


# name -> make(): the model, sizes(model): [(input size, rows)], rounding: sizes with the tier-2 pass (None: all)
CONFIGS = {
    'resnet20_cifar': _cifar('resnet', 64, depth=20),
    'resnet44_cifar': _cifar('resnet', 64, depth=44),
    'resnet44_cifar_sampled': dict(_cifar('resnet', 0, depth=44, regime='sampled_D+'), sizes=_sampled),
    'wrn28_10_dropout': _cifar('resnet', 128, depth=28, width=[160, 320, 640], regime='wide-resnet', dropout=0.3),
    'resnext20_cifar': _cifar('resnext', 64, depth=20),
    'resnet20_cifar_l1': _cifar('resnet', 64, depth=20, bn_norm='L1'),
    'resnet50_sampled': dict(_imagenet('resnet', 0, depth=50, regime='sampled_D+'), sizes=_sampled),
    'resnet50_sampled144': dict(_imagenet('resnet', 0, depth=50, regime='sampled_D+144'), sizes=_sampled),
    'resnet18': _imagenet('resnet', 32, depth=18),
    'resnet18_l1': _imagenet('resnet', 32, depth=18, bn_norm='L1'),
    'resnext50': _imagenet('resnext', 32, depth=50),
    'resnext101': _imagenet('resnext', 32, depth=101),
    'resnet_se50': _imagenet('resnet_se', 32, depth=50),
    'resnext_se50': _imagenet('resnext_se', 32, depth=50),
    'mobilenet_v2': _imagenet('mobilenet_v2', 32),
    'mobilenet_v1': _imagenet('mobilenet', 32),
}
_ROUNDING = [n for n, c in CONFIGS.items() if c['rounding'] is None or 224 in c['rounding']]


# ------------------------------------------------------------------------------------------------ recorder
class _Recorder(object):
    """wraps every public function of ops while installed: conv calls become signatures, the others (name, shapes)"""

    def __init__(self, ops):
        self.ops = ops
        self.convs = []        # dicts: dir, desc, flags, operand pointers, groups info
        self.calls = []        # (name, tensor shapes) of every other entry point
        self.packs = {}        # output pointer of group_weight_pack -> (K, T, C, groups, window, transpose)
        self.keep = []         # packed operands and windowed gradients stay alive: their pointers stay unique
        self.saved = {}

    def __enter__(self):
        for name, fn in vars(self.ops).items():
            if name.startswith('_') or not inspect.isfunction(fn) or fn.__module__ != self.ops.__name__:
                continue
            self.saved[name] = fn
            setattr(self.ops, name, self._wrap(name, fn))
        return self

    def __exit__(self, *exc):
        for name, fn in self.saved.items():
            setattr(self.ops, name, fn)

    def _wrap(self, name, fn):
        sig = inspect.signature(fn)

        def wrapper(*a, **kw):
            out = fn(*a, **kw)
            self._note(name, sig.bind(*a, **kw).arguments, out)
            return out
        return wrapper

    def _note(self, name, args, out):
        if name in CONV:
            d = args['desc']
            r = dict(dir=DIRS[name], desc=tuple(int(getattr(d, f)) for f in DESC_FIELDS), group=None,
                     bias=args.get('bias') is not None, res=args.get('residual') is not None,
                     act=int(args.get('act', 0)), fp32=bool(args.get('out_fp32', False)),
                     stats=args.get('bn_stats_ws') is not None)
            w = args['w'] if name == 'conv_fprop' else (args['wt'] if name == 'conv_dgrad' else args['dw'])
            r['operand'] = (w.data_ptr(), w.numel())
            if name != 'conv_wgrad':
                r['group'] = self.packs.get(w.data_ptr())
            self.convs.append(r)
        elif name == 'group_weight_pack':
            self.packs[out.data_ptr()] = (args['K'], args['T'], args['C'], args['groups'], args['window'],
                                          bool(args.get('transpose', False)))
            self.keep.append(out)
        elif name == 'group_wgrad_unpack':
            dw = args['dw_win']
            hit = [r for r in self.convs if r['dir'] == 'w' and r['operand'][0] == dw.data_ptr()]
            if hit:
                hit[-1]['group'] = (args['K'], args['T'], args['C'], args['groups'], args['window'], False)
            self.keep.append(dw)
        self.calls.append((name, {k: tuple(v.shape) for k, v in args.items() if torch.is_tensor(v)}))


def _case_of(r):
    """the sweep case of one recorded conv call; raises ValueError when the call does not map onto one"""
    d = dict(zip(DESC_FIELDS, r['desc']))
    T = d['R'] * d['S']
    wgrad = r['dir'] == 'w'
    if r['group'] is not None:
        K, t, C, groups, window, transpose = r['group']
        if (K, t, C) != (d['K'], T, d['C']) or transpose != (r['dir'] == 'd') or window != (d['window'] or C):
            raise ValueError('grouped operand %s does not belong to descriptor %s' % (r['group'], d))
    else:
        groups = 1
        if d['window'] or r['operand'][1] != d['K'] * T * d['C']:
            raise ValueError('operand of %d elements for an ungrouped descriptor %s' % (r['operand'][1], d))
    xs = (d['x_pixel_stride'], d['x_row_stride'], d['x_image_stride'])
    try:
        cs = cs_sweep._case(d['N'], d['H'], d['W'], d['C'], d['K'], d['R'], d['S'], d['stride'],
                            (d['pad_h'], d['pad_w']), ops=r['dir'], bias=r['bias'], act=r['act'], fp32=r['fp32'],
                            stats=r['stats'], groups=groups, window=64 if d['window'] else 0,
                            x_strides=xs if any(xs) else None, res_f=r['res'] and r['dir'] == 'f',
                            res_d=r['res'] and r['dir'] == 'd', P=d['P'], Q=d['Q'])
    except AssertionError as e:
        raise ValueError('%s: %s' % (d, e))
    again = cs_sweep._desc(cs, wgrad=wgrad)
    if tuple(int(getattr(again, f)) for f in DESC_FIELDS) != r['desc']:
        raise ValueError('the case does not reproduce descriptor %s' % d)
    return cs


def _signature(r, cs):
    g = cs['groups']
    return (r['dir'],) + r['desc'] + (g, r['bias'], r['res'], r['act'], r['fp32'], r['stats'])


def _tag(sig):
    return 'census ' + ' '.join(str(v) for v in sig)


def _record(name):
    """-> {'cases': {signature: case}, 'origins': {signature: {(config, size)}}, 'unmapped', 'unlisted', 'bn'}"""
    from convnet.pytorch_b200 import engine, ops
    cfg = CONFIGS[name]
    torch.manual_seed(0)
    model = cfg['make']()
    out = dict(cases={}, origins={}, unmapped=[], unlisted=set(), bn=set(), sizes=[], dirs={})
    with _Recorder(ops) as rec0:
        engine.convert_b200(model, 'cuda')
    rt = model._b200
    saved = engine.FOLD_BN_EVAL
    try:
        for size, rows in cfg['sizes'](model):
            out['sizes'].append((size, rows))
            g = torch.Generator().manual_seed(size * 1000 + rows)
            x = torch.randn(rows, 3, size, size, generator=g).cuda()
            y = torch.randint(0, rt.classes, (rows,), generator=g).cuda()
            with _Recorder(ops) as rec:
                model.train()
                rt.train_step(x, y)
                model.eval()
                with torch.no_grad():
                    for fold in (True, False):
                        engine.FOLD_BN_EVAL = fold
                        model(x)
                torch.cuda.synchronize()
            for r in rec.convs:
                try:
                    cs = _case_of(r)
                except ValueError as e:
                    out['unmapped'].append('%s @%d px: %s' % (r['dir'], size, e))
                    continue
                sig = _signature(r, cs)
                out['cases'].setdefault(sig, cs)
                out['origins'].setdefault(sig, set()).add((name, size))
            for call, shapes in rec0.calls + rec.calls:
                if call not in CONV and call not in ('group_weight_pack', 'group_wgrad_unpack') and \
                        call not in ELSEWHERE:
                    out['unlisted'].add(call)
                if call in BN_FAMILY:
                    z = shapes['z']
                    out['bn'].add((math.prod(z) // z[-1], z[-1]))
            del rec
    finally:
        engine.FOLD_BN_EVAL = saved
    for sig in out['cases']:
        out['dirs'][sig[0]] = out['dirs'].get(sig[0], 0) + 1
    del model, rt
    torch.cuda.empty_cache()
    return out


_RECORDS = {}
PASSED = {}        # signature -> tag: the unique cases that passed the exact tier
ROUNDED = set()
BN_DONE = set()
WORST = {}         # tier-2 output type -> (worst ratio, where)
SECONDS = {}       # (config, what) -> wall seconds


def recording(name):
    if name not in _RECORDS:
        t0 = time.time()
        _RECORDS[name] = _record(name)
        SECONDS[(name, 'record')] = time.time() - t0
    return _RECORDS[name]


def _checked(name):
    rec = recording(name)
    assert not rec['unmapped'], '%s: convolution calls that map onto no sweep case: %s' % (name, rec['unmapped'][:5])
    assert not rec['unlisted'], '%s: ops entry points missing from ELSEWHERE: %s' % (name, sorted(rec['unlisted']))
    for d in 'fdw':
        assert rec['dirs'].get(d, 0) > 0, '%s: no %s convolution recorded' % (name, d)
    return rec


def _run_exact(name):
    rec = _checked(name)
    t0 = time.time()
    for i, (sig, cs) in enumerate(rec['cases'].items()):
        if sig not in PASSED:
            cs_sweep.check_exact(cs, _tag(sig), rng='cuda')
            PASSED[sig] = _tag(sig)
        if i % 40 == 39:
            print('census %s: %d of %d exact, %.1f s' % (name, i + 1, len(rec['cases']), time.time() - t0), flush=True)
    SECONDS[(name, 'exact')] = SECONDS.get((name, 'exact'), 0) + time.time() - t0
    print('census %s: %d unique convolutions, exact tier %.1f s' % (name, len(rec['cases']), time.time() - t0))
    return rec


# ------------------------------------------------------------------------------------------------ tests
@pytest.mark.parametrize('name', list(CONFIGS))
def test_census_exact(name):
    """every unique convolution of the configuration, tier 1 (bit for bit against fp64) at the real batch"""
    _run_exact(name)


@pytest.mark.parametrize('name', _ROUNDING)
def test_census_rounding(name):
    """tier 2 (rounding bounds) for the unique convolutions of the CIFAR configurations and of 224 px"""
    rec = _checked(name)
    sizes = CONFIGS[name]['rounding']
    t0 = time.time()
    for sig, cs in rec['cases'].items():
        if sig in ROUNDED or not any(sizes is None or s in sizes for _, s in rec['origins'][sig]):
            continue
        cs_sweep.check_rounding(cs, _tag(sig), WORST, rng='cuda', coef=COEF)
        ROUNDED.add(sig)
    SECONDS[(name, 'rounding')] = time.time() - t0
    print('census %s: rounding tier %.1f s' % (name, time.time() - t0))


@pytest.mark.parametrize('name', list(CONFIGS))
def test_census_batchnorm(name):
    """the kernel sweep's tier-1 BatchNorm checks at every recorded (M, C) whose C is outside its channel list"""
    rec = _checked(name)
    t0 = time.time()
    for M, C in sorted(rec['bn']):
        if C in k_sweep.BN_CS or (M, C) in BN_DONE:
            continue
        tag = 'census M=%d C=%d' % (M, C)
        k_sweep.check_bn_stats(M, C, 1, tag, rng='cuda')
        k_sweep.check_bn_apply(M, C, 1, tag, rng='cuda')
        k_sweep.check_bn_backward(M, C, 1, tag, rng='cuda')
        BN_DONE.add((M, C))
    SECONDS[(name, 'batchnorm')] = time.time() - t0
    print('census %s: BatchNorm checks %.1f s' % (name, time.time() - t0))


def _witnesses():
    """label -> predicate over debug-line records of exact-tier-passed census cases"""
    igd1 = lambda r: r['kind'] == 'igemm' and r['op'] == 'dgrad' and r['filt'] == (1, 1) and r['res']
    folded = lambda r: r['op'] == 'fprop' and r['bias'] and r['res'] and r['act'] == 1
    stem = lambda r, px: r['cs']['K'] == 64 and r['cs']['H'] == px // 2 + 3 and r['op'] == 'fprop'
    mm16 = lambda r: ('resnet44_cifar_sampled', 16) in r['origins'] and r['cs']['K'] == 64 and r['cs']['R'] == 3
    w = {'1x1 dgrad + residual, Nout = %d' % n: (lambda r, n=n: igd1(r) and r['N'] == n) for n in (24, 32, 96, 160)}
    w.update({
        '1x1 dgrad + residual, Nout = 256': lambda r: igd1(r) and r['N'] == 256,
        'folded bias + residual + ReLU on the halo kernel': lambda r: r['kind'] == 'halo' and folded(r),
        'folded bias + residual + ReLU on igemm': lambda r: r['kind'] == 'igemm' and folded(r),
        '128 px stem on igemm, taps = 16, C = 16':
            lambda r: stem(r, 128) and r['kind'] == 'igemm' and r['taps'] == 16 and r['C'] == 16,
        '320 px wide-pixel stem': lambda r: stem(r, 320) and r['kind'] == 'igemm' and r['xs'] > 0,
        '96 px stem on the halo kernel': lambda r: stem(r, 96) and r['kind'] == 'halo' and r['taps'] == 16,
        'igemm block_n 80': lambda r: r['kind'] == 'igemm' and r['block_n'] == 80,
        '3x3 stride 1 at 640 channels on igemm (the halo kernel refuses them)':
            lambda r: r['kind'] == 'igemm' and r['filt'] == (3, 3) and r['conv_stride'] == 1 and r['N'] == 640,
        'Mix&Match 16 px layer-3 fprop on igemm': lambda r: mm16(r) and r['kind'] == 'igemm' and r['op'] == 'fprop',
        'Mix&Match 16 px layer-3 dgrad on igemm': lambda r: mm16(r) and r['kind'] == 'igemm' and r['op'] == 'dgrad',
        'Mix&Match 16 px layer-3 wgrad': lambda r: mm16(r) and r['kind'] == 'wgrad',
    })
    return w


def test_census_witnesses_and_report(monkeypatch, capfd):
    """The shapes the census exists for are recorded and passed the exact tier; prints the census."""
    t_start = time.time()
    cases, origins = {}, {}
    for name in CONFIGS:
        rec = _run_exact(name)
        for sig, c in rec['cases'].items():
            cases.setdefault(sig, c)
            origins.setdefault(sig, set()).update(rec['origins'][sig])
    cs_sweep.enable_debug_lines(monkeypatch)
    by_tag = {_tag(sig): sig for sig in cases}
    recs = cs_sweep.coverage_records({_tag(sig): c for sig, c in cases.items() if sig in PASSED}, capfd)
    for r in recs:
        sig = by_tag[r['case']]
        r['cs'], r['origins'] = cases[sig], origins[sig]
    sweep_recs = cs_sweep.coverage_records(cs_sweep.sweep(cs_sweep._sm_count()), capfd)
    lines = ['census: %d unique convolutions' % len(cases)]
    for name in CONFIGS:
        rec = _RECORDS[name]
        lines.append('  %-24s sizes %-40s fprop %3d  dgrad %3d  wgrad %3d  BN shapes %3d' % (
            name, ' '.join('%d@%d' % sr for sr in rec['sizes']), rec['dirs'].get('f', 0), rec['dirs'].get('d', 0),
            rec['dirs'].get('w', 0), len(rec['bn'])))
    missing = []
    for label, pred in _witnesses().items():
        hit = next((r for r in recs if pred(r)), None)
        if hit is None:
            missing.append(label)
        else:
            lines.append('witness: %-50s %s' % (label, hit['case']))
    req = cs_sweep._requirements()
    new = [label for label, pred in req.items() if any(pred(r) for r in recs) and not any(pred(r) for r in sweep_recs)]
    lines.append('kernel configurations reached by the census and not by the sweep: %s' % (new or 'none'))
    lines.append('igemm block_n reached: %s' % sorted({r['block_n'] for r in recs if r['kind'] == 'igemm'}))
    for key, c in zip(('bf16', 'fp32'), COEF[:2]):
        if key in WORST:
            ratio, where = WORST[key]
            lines.append('tier-2 %s outputs: worst (|y-ref| - rt|ref|)/absref = %.3e (%s), bound %.3e (%.1fx)' % (
                key, ratio, where, c, c / ratio if ratio > 0 else math.inf))
    SECONDS[('all', 'witnesses')] = time.time() - t_start
    for (name, what), s in sorted(SECONDS.items()):
        lines.append('seconds: %-24s %-10s %8.1f' % (name, what, s))
    lines.append('seconds in this session: %.1f' % sum(SECONDS.values()))
    with capfd.disabled():
        print('\n' + '\n'.join(lines))
    assert not missing, 'census witnesses not reached: %s' % missing
