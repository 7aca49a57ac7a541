"""Per-launch GPU time table of one steady-state cfg-2 frame (warm caches, eager launches bracketed
by CUDA events; each bracket includes the launch gap, so small kernels read a few us high)."""
import sys, os, collections
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import mivos_b200
from mivos_b200 import ops, synth

torch.set_grad_enabled(False)
dev = torch.device("cuda:0")
net = mivos_b200.PropagationNetwork(top_k=20)
net.load_state_dict(synth.make_prop_state_dict())
net = net.to(dev)
K, T, hw = 1, 20, 30 * 54
frame = torch.randn(1, 3, 480, 864, device=dev)
bank_k = torch.randn((K, (T + 1) * hw, 128), device=dev)
bank_v = torch.randn((K, (T + 1) * hw, 512), device=dev)
rec = []
names = ["conv_gemm", "stem_gather", "gather_s2", "maxpool3x3s2", "upsample2x_add", "halo_copy", "memory_read",
         "upsample4x_sigmoid_aggregate", "bank_write", "halo_to_pixels"]
orig = {n: getattr(ops, n) for n in names}


def wrap(n):
    f = orig[n]

    def g(*a, **k):
        e0, e1 = torch.cuda.Event(True), torch.cuda.Event(True)
        e0.record()
        r = f(*a, **k)
        e1.record()
        if n == "conv_gemm":
            x, pc, nn, h, w = a[:5]
            sig = f"conv {pc.ksize}x{pc.ksize}/{pc.stride} {pc.cin}->{pc.cout} @{h}x{w} n={nn}"
            fl = 2.0 * nn * h * w * pc.ksize ** 2 * pc.cin * pc.cout
        else:
            sig, fl = n, 0.0
        rec.append((sig, e0, e1, fl))
        return r
    return g


def frame_step(qs):
    qs = net.encode_query_resident(frame, qs)
    _, prob = net.engine().segment(bank_k, bank_v, T * hw, qs, K)
    net.memorize_resident(frame, prob[1:], bank_k, bank_v, T)
    return qs


qs = None
for _ in range(3):
    qs = frame_step(qs)
for n in names:
    setattr(ops, n, wrap(n))
reps = 5
for _ in range(reps):
    qs = frame_step(qs)
torch.cuda.synchronize()
agg = collections.OrderedDict()
for sig, e0, e1, fl in rec:
    a = agg.setdefault(sig, [0, 0.0, 0.0])
    a[0] += 1
    a[1] += e0.elapsed_time(e1) * 1e3
    a[2] += fl
tot = sum(a[1] for a in agg.values()) / reps
print(f"frame total (sum of bracketed launches): {tot:.0f} us over {len(rec)//reps} launches")
for sig, (c, us, fl) in sorted(agg.items(), key=lambda kv: -kv[1][1]):
    print(f"{us/reps:8.1f} us/frame  n={c//reps:2d}  {us/c:7.1f} us each  {fl/us/1e6 if fl else 0:7.1f} TF/s  {sig}")
