"""Per-layer roofline fractions from a tools/layer_bench.py log: t_roof = max(FLOPs / P_tensor, bytes / BW_hbm) with the
H100 SXM data-sheet peaks (989 TFLOP/s dense bf16, 3.35 TB/s HBM3 at 700 W), bytes = input + output (+ residual) once in
bf16 + weights.   usage: layer_roofline.py layer_bench.log"""
import json
import sys

B = 256
LAYERS = {  # name: (H, C, K, R, stride, pad)  -- same table as tools/layer_bench.py
    'stem_halo_4x4': (115, 16, 64, 4, 1, 0), 'l1_1x1_64_64': (56, 64, 64, 1, 1, 0), 'l1_3x3_64_64': (56, 64, 64, 3, 1, 1),
    'l1_1x1_64_256': (56, 64, 256, 1, 1, 0), 'l1_1x1_256_64': (56, 256, 64, 1, 1, 0),
    'l2_1x1_256_128': (56, 256, 128, 1, 1, 0), 'l2_3x3s2_128_128': (56, 128, 128, 3, 2, 1),
    'l2_1x1_128_512': (28, 128, 512, 1, 1, 0), 'l2_ds_256_512_s2': (56, 256, 512, 1, 2, 0),
    'l2_1x1_512_128': (28, 512, 128, 1, 1, 0), 'l2_3x3_128_128': (28, 128, 128, 3, 1, 1),
    'l3_3x3_256_256': (14, 256, 256, 3, 1, 1), 'l3_1x1_256_1024': (14, 256, 1024, 1, 1, 0),
    'l3_1x1_1024_256': (14, 1024, 256, 1, 1, 0), 'l4_3x3_512_512': (7, 512, 512, 3, 1, 1),
    'l4_1x1_512_2048': (7, 512, 2048, 1, 1, 0), 'l4_1x1_2048_512': (7, 2048, 512, 1, 1, 0),
}


P, BW = 989e12, 3350e9


def main(log):
    print('| layer | pass | measured us | roofline us (bound) | fraction |')
    print('|---|---|---:|---:|---:|')
    tot_m = tot_r = 0.0
    for line in open(log):
        name, _, js = line.partition(' ')
        if name not in LAYERS:
            continue
        H, C, K, R, stride, pad = LAYERS[name]
        Po = (H + 2 * pad - R) // stride + 1
        flops = 2.0 * B * Po * Po * K * R * R * C
        x_b, y_b, w_b = B * H * H * C * 2, B * Po * Po * K * 2, K * R * R * C * 2
        res = json.loads(js.strip())
        for kind, extra in (('fprop', 0), ('dgrad', 0), ('dgrad_res', x_b), ('wgrad', 0)):
            r = res.get(kind)
            if not isinstance(r, dict):
                continue
            nbytes = x_b + y_b + w_b + extra + (w_b if kind == 'wgrad' else 0)   # wgrad writes fp32 dw
            t_t, t_b = flops / P, nbytes / BW
            t_roof = max(t_t, t_b) * 1e6
            tot_m += r['us']; tot_r += t_roof
            print('| %s | %s | %.0f | %.0f (%s) | %.2f |' % (name, kind, r['us'], t_roof, 'tensor' if t_t > t_b else 'hbm',
                                                         t_roof / r['us']))
    print('| **all listed** | | %.0f | %.0f | %.2f |' % (tot_m, tot_r, tot_r / tot_m))


if __name__ == '__main__':
    main(*sys.argv[1:])
