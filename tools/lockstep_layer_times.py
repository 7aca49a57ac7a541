"""Per-launch GPU time table of the unit the headline bench times: one lock-step step of C clips
(segment + encode_memory at C clips + bank writes, cfg-2 shapes, 20-frame bank) plus the batched
query pass of 8 frames, eager launches bracketed by CUDA events, reported per CLIP-FRAME.
usage: python tools/lockstep_layer_times.py [C=4] [fp16|tf32]"""
import sys, os, collections
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import mivos_b200
from mivos_b200 import ops, synth

C = int(sys.argv[1]) if len(sys.argv) > 1 else 4
act = torch.float32 if (len(sys.argv) > 2 and sys.argv[2] == "tf32") else torch.float16
torch.set_grad_enabled(False)
dev = torch.device("cuda:0")
net = mivos_b200.PropagationNetwork(top_k=20, act_dtype=act)
net.load_state_dict(synth.make_prop_state_dict())
net = net.to(dev)
eng = net.engine()
K, T, H, W = 1, 20, 480, 864
hw = (H // 16) * (W // 16)
QN = 8
frames_q = torch.randn(QN, 3, H, W, device=dev)
frames = torch.randn(C, 3, H, W, device=dev)
bank_k = torch.randn((C * K, (T + 1) * hw, 128), device=dev)
bank_v = torch.randn((C * K, (T + 1) * hw, 512), device=dev)
prob = torch.zeros((C, K + 1, 1, H, W), device=dev)
_, qbatch8 = eng.new_query_states(H, W, QN)
_, qbatch = eng.new_query_states(H, W, C)
rec = []
names = ["conv_gemm", "stem_gather", "gather_s2", "maxpool3x3s2", "upsample2x_add", "halo_copy", "memory_read",
         "upsample4x_sigmoid_aggregate", "bank_write", "halo_to_pixels"]
orig = {n: getattr(ops, n) for n in names}
phase = ["?"]


def wrap(n):
    f = orig[n]

    def g(*a, **k):
        e0, e1 = torch.cuda.Event(True), torch.cuda.Event(True)
        e0.record()
        r = f(*a, **k)
        e1.record()
        if n == "conv_gemm":
            x, pc, nn, h, w = a[:5]
            sig = f"conv {pc.ksize}x{pc.ksize}/{pc.stride} {pc.cin}->{pc.cout} @{h}x{w} n={nn}" + (" +res" if k.get("residual") is not None else "")
            fl = 2.0 * nn * h * w * pc.ksize ** 2 * pc.cin * pc.cout
        else:
            sig, fl = n, 0.0
        rec.append((phase[0] + " " + sig, e0, e1, fl, phase[0]))
        return r
    return g


def query_pass():
    phase[0] = "Q"
    eng.encode_query_batch(frames_q, qbatch8)


def step():
    phase[0] = "S"
    eng.segment(bank_k, bank_v, T * hw, qbatch, K, C, prob_out=prob)
    phase[0] = "M"
    kv = eng.encode_memory(frames, prob[:, 1:])
    for c in range(C):
        o = slice(c * K, (c + 1) * K)
        ops.bank_write(kv[o], K, H // 16, W // 16, 0, 128, bank_k[o], bank_v[o], T)


eng.encode_query_batch(frames[:C], qbatch)
for _ in range(2):
    query_pass()
    step()
for n in names:
    setattr(ops, n, wrap(n))
reps = 3
for _ in range(reps):
    query_pass()
    step()
torch.cuda.synchronize()
agg = collections.OrderedDict()
ph_tot = collections.OrderedDict()
for sig, e0, e1, fl, ph in rec:
    div = QN if ph == "Q" else C  # per clip-frame
    us = e0.elapsed_time(e1) * 1e3
    a = agg.setdefault(sig, [0, 0.0, 0.0, div])
    a[0] += 1
    a[1] += us
    a[2] += fl
    p = ph_tot.setdefault(ph, [0.0, 0.0, 0])
    p[0] += us / div
    p[1] += fl / div
    p[2] += 1
print(f"lock-step C={C} (+ query pass N={QN}), {'fp16' if act == torch.float16 else 'tf32'}; all figures per CLIP-FRAME")
for ph, (us, fl, n) in ph_tot.items():
    print(f"phase {ph}: {us/reps:8.1f} us/clip-frame, {fl/reps/1e9:7.1f} GFLOP conv, {n//reps} launches/pass")
tot = sum(p[0] for p in ph_tot.values()) / reps
print(f"total (sum of bracketed launches): {tot:.0f} us per clip-frame")
for sig, (c, us, fl, div) in sorted(agg.items(), key=lambda kv: -kv[1][1] / kv[1][3]):
    print(f"{us/reps/div:8.1f} us/clip-frame  n={c//reps:2d}  {us/c:7.1f} us each  {fl/us/1e6 if fl else 0:7.1f} TF/s  {sig}")
