"""Per-tensor gradient comparison of the kernel pipeline against the bf16-emulating CPU oracle (diagnostic)."""
import sys, os, copy
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import torch.nn.functional as F
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'tests'))
from test_gpu_engine import _pair, _rel, _cos
from convnet.pytorch_b200.models import resnet
from oracle import ref_model

depth = int(sys.argv[1]) if len(sys.argv) > 1 else 18
size = int(sys.argv[2]) if len(sys.argv) > 2 else 64
batch = int(sys.argv[3]) if len(sys.argv) > 3 else 8
cfg = dict(dataset='imagenet', depth=depth) if depth != 20 else dict(dataset='cifar10', depth=20)
classes = 1000 if depth != 20 else 10
ref, mine, x, y = _pair(resnet, cfg, (3, size, size), classes, batch=batch)
sd = {k: v.detach().cpu().clone() for k, v in ref.state_dict().items()}
mine.train(); mine._b200.arena.zero_grad()
lo = mine(x); loss = F.cross_entropy(lo, y); loss.backward(); torch.cuda.synchronize()
for quant in (True, False):
    ol, oloss, og, ob = ref_model.loss_and_grads(sd, x.cpu(), y.cpu(), quant=quant)
    print('quant=%s logits rel %.3e loss %.5f vs %.5f' % (quant, _rel(lo.cpu(), ol), float(loss), float(oloss)))
    rows = []
    for n, p in mine.named_parameters():
        if float(og[n].norm()) > 0:
            rows.append((_rel(p.grad.cpu(), og[n]), _cos(p.grad.cpu(), og[n]), float(og[n].norm()), n))
    gm = torch.cat([p.grad.cpu().flatten() for _, p in mine.named_parameters()])
    go = torch.cat([og[n].flatten() for n, _ in mine.named_parameters()])
    print('  global rel %.3e cos %.5f' % (_rel(gm, go), _cos(gm, go)))
    rows.sort(reverse=True)
    for r in rows[:12]:
        print('  rel %.3e cos %.5f norm %.3e %s' % r)
    print('  ... best:')
    for r in rows[-4:]:
        print('  rel %.3e cos %.5f norm %.3e %s' % r)
