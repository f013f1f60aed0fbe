"""Per-layer timing of the conv kernels on ResNet-50 shapes (batch 256): CUDA-event median per launch, achieved
TFLOP/s and algorithmic GB/s.  usage: layer_bench.py [filter] [--once]   (--once: one launch each)"""
import sys, os, json
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from convnet.pytorch_b200 import ops

B = 256
# name: (H, C, K, R, stride, pad)
LAYERS = {
    'stem_s2d_4x4':     (112, 16, 64, 4, 1, 2),
    'stem_halo_4x4':    (115, 16, 64, 4, 1, 0),
    'l1_1x1_64_64':     (56, 64, 64, 1, 1, 0),
    'l1_3x3_64_64':     (56, 64, 64, 3, 1, 1),
    'l1_1x1_64_256':    (56, 64, 256, 1, 1, 0),
    'l1_1x1_256_64':    (56, 256, 64, 1, 1, 0),
    'l2_1x1_256_128':   (56, 256, 128, 1, 1, 0),
    'l2_3x3s2_128_128': (56, 128, 128, 3, 2, 1),
    'l2_1x1_128_512':   (28, 128, 512, 1, 1, 0),
    'l2_ds_256_512_s2': (56, 256, 512, 1, 2, 0),
    'l2_1x1_512_128':   (28, 512, 128, 1, 1, 0),
    'l2_3x3_128_128':   (28, 128, 128, 3, 1, 1),
    'l3_3x3_256_256':   (14, 256, 256, 3, 1, 1),
    'l3_1x1_256_1024':  (14, 256, 1024, 1, 1, 0),
    'l3_1x1_1024_256':  (14, 1024, 256, 1, 1, 0),
    'l4_3x3_512_512':   (7, 512, 512, 3, 1, 1),
    'l4_1x1_512_2048':  (7, 512, 2048, 1, 1, 0),
    'l4_1x1_2048_512':  (7, 2048, 512, 1, 1, 0),
}


def run(name, kinds, once):
    H, C, K, R, stride, pad = LAYERS[name]
    P = None
    if name == 'stem_halo_4x4':
        desc = ops.make_desc(B, H, H, C, K, R, R, stride, pad)
    elif name.startswith('stem'):
        desc = ops.make_desc(B, H, H, C, K, R, R, stride, pad, P=H, Q=H)
    else:
        desc = ops.make_desc(B, H, H, C, K, R, R, stride, pad)
    x = torch.randn(B, H, H, C, device='cuda').to(torch.bfloat16)
    w = torch.randn(K, R * R, C, device='cuda').to(torch.bfloat16) * 0.05
    wt = ops.weight_transpose(w)
    dy = torch.randn(B, desc.P, desc.Q, K, device='cuda').to(torch.bfloat16)
    res = torch.randn(B, H, H, C, device='cuda').to(torch.bfloat16)
    dw = torch.zeros(K, R * R, C, device='cuda')
    y = torch.empty(B, desc.P, desc.Q, K, device='cuda', dtype=torch.bfloat16)
    dx = torch.empty(B, H, H, C, device='cuda', dtype=torch.bfloat16)
    flops = 2.0 * B * desc.P * desc.Q * K * R * R * C
    in_b, out_b = x.numel() * 2, y.numel() * 2
    fns = {'fprop': (lambda: ops.conv_fprop(x, w, desc, out=y), in_b + out_b),
           'dgrad': (lambda: ops.conv_dgrad(dy, wt, desc, out=dx), in_b + out_b),
           'dgrad_res': (lambda: ops.conv_dgrad(dy, wt, desc, out=dx, residual=res), 2 * in_b + out_b),
           'wgrad': (lambda: ops.conv_wgrad(x, dy, desc, dw), in_b + out_b)}
    flush = torch.empty(256 * 1024 * 1024, device='cuda', dtype=torch.uint8)
    out = {}
    for kind in kinds:
        if kind.startswith('dgrad') and name.startswith('stem'):
            continue
        fn, nbytes = fns[kind]
        try:
            fn(); torch.cuda.synchronize()
        except Exception as e:
            out[kind] = 'unsupported'
            continue
        if once:
            continue
        for _ in range(2):
            fn()
        ts = []
        for _ in range(5):
            flush.zero_()           # evict L2 between timed launches
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(); fn(); e1.record(); torch.cuda.synchronize()
            ts.append(e0.elapsed_time(e1))
        ts.sort()
        ms = ts[len(ts) // 2]
        out[kind] = {'us': round(ms * 1e3, 1), 'tflops': round(flops / ms / 1e9, 1), 'gbs': round(nbytes / ms / 1e6, 0)}
    return out


if __name__ == '__main__':
    args = [a for a in sys.argv[1:] if not a.startswith('--')]
    once = '--once' in sys.argv
    kinds = ['fprop', 'dgrad', 'dgrad_res', 'wgrad']
    for a in list(args):
        if a in kinds:
            kinds = [a]; args.remove(a)
    filt = args[0] if args else ''
    for name in LAYERS:
        if filt in name:
            r = run(name, kinds, once)
            if not once:
                print('%-18s %s' % (name, json.dumps(r)))
