"""Which tensors carry the gradient error?  usage: parity_diag.py <depth> <size> <batch> [oracle]
Prints, for the kernel pipeline vs stock torch fp32 (and vs the bf16-storage CPU oracle with `oracle`), the tensors sorted
by their share of the squared global gradient error."""
import sys, os, copy
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'tests'))
import torch
import torch.nn.functional as F
from test_gpu_engine import _pair, _rel, _cos

depth, size, batch = int(sys.argv[1]), int(sys.argv[2]), int(sys.argv[3])
from convnet.pytorch_b200.models import resnet
cfg = dict(dataset='imagenet', depth=depth) if size > 32 else dict(dataset='cifar10', depth=depth)
ref, mine, x, y = _pair(resnet, cfg, (3, size, size), 1000 if size > 32 else 10, steps=5, batch=batch)
ref.train(); mine.train()
xq = x.to(torch.bfloat16).float()
ref.zero_grad(); F.cross_entropy(ref(xq), y).backward()
mine._b200.arena.zero_grad(); lo = mine(x); F.cross_entropy(lo, y).backward()
torch.cuda.synchronize()
pm, pr = dict(mine.named_parameters()), dict(ref.named_parameters())


def report(tag, other):
    tot_err = sum(float((pm[n].grad.double().cpu() - other[n].double().cpu()).pow(2).sum()) for n in pm)
    tot = sum(float(other[n].double().pow(2).sum()) for n in pm)
    print('== %s: global rel %.3e' % (tag, (tot_err / tot) ** 0.5))
    rows = []
    for n in pm:
        a, b = pm[n].grad.double().cpu(), other[n].double().cpu()
        e = float((a - b).pow(2).sum())
        rows.append((e / tot_err, float(b.pow(2).sum()) / tot, _cos(a, b), _rel(a, b), n))
    for r in sorted(rows, reverse=True)[:12]:
        print('  err share %.3f  norm share %.3f  cos %.5f  rel %.3e  %s' % r)


report('vs torch fp32', {n: p.grad for n, p in pr.items()})
if len(sys.argv) > 4:
    from oracle import ref_model
    sd = {k: v.detach().cpu().clone() for k, v in ref.state_dict().items()}
    o_logits, o_loss, o_grads, _ = ref_model.loss_and_grads(sd, x.cpu(), y.cpu(), quant=True)
    print('logits vs oracle %.3e' % _rel(lo.cpu(), o_logits))
    report('vs bf16 oracle', o_grads)
    tot_err = sum(float((o_grads[n].double() - pr[n].grad.double().cpu()).pow(2).sum()) for n in pm)
    tot = sum(float(pr[n].grad.double().pow(2).sum()) for n in pm)
    print('== oracle-bf16 vs torch fp32 (the ideal pipeline own drift): global rel %.3e' % ((tot_err / tot) ** 0.5))
