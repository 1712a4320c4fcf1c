"""Debug helper: per-phase cycle breakdown of the warp-tiled decode kernel (needs a GPU)."""
import sys, ctypes, torch, numpy as np
sys.path.insert(0, '.'); sys.path.insert(0, '..')
from bench import make_model
from pytorchwavenetvocoder_b200 import _lib
lib = _lib.load()
dev = torch.device('cuda')
cfg, net = make_model(dev, 'fp32'); net.eval()
B, n = int(sys.argv[1]) if len(sys.argv) > 1 else 64, 2000
buf = torch.zeros(2 * B * 16, dtype=torch.int64, device=dev)   # (2 CTAs per utterance in the cluster form)
lib.wnb_decode_warp_set_timing(ctypes.c_void_p(buf.data_ptr()))
h = torch.randn(B, 28, (n + 80) // 80, device=dev); x = torch.full((B, 1), 128, dtype=torch.int64, device=dev)
with torch.no_grad():
    net._decode(x, h, [n] * B, 'sampling', seed=1)
torch.cuda.synchronize()
lib.wnb_decode_warp_set_timing(None)
t = buf.view(-1, 16).cpu().numpy().astype(np.float64)
t = t[t.sum(1) > 0]
names = ['prologue', 'sync0', 'gateGEMV', 'reduce+gate', 'sync1', 'resGEMV', 'skipGEMV', 'sync2', 'post1', 'post2', 'pick']
per = t.mean(0)[:11] / n
print('kernel:', net.last_decode_kernel, ' CTAs', len(t), ' cycles/step total %.0f' % per.sum())
print('  blocked in acquire() (warp 0): %.0f cyc/step' % (t.mean(0)[12] / n))
for k, v in zip(names, per):
    print('  %-12s %9.0f cyc/step  %5.1f%%' % (k, v, 100 * v / per.sum()))
