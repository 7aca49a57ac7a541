"""Phase timings at cfg-2 shapes: batched query pass for N = 1, 2, 4, 8 frames, and the sequential
per-frame step (memory read + decoder tail + memorize) eager vs CUDA-graph replay."""
import sys, os, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import mivos_b200
from mivos_b200 import synth, _lib
from mivos_b200.frame_step import FrameStep

torch.set_grad_enabled(False)
dev = torch.device("cuda:0")
net = mivos_b200.PropagationNetwork(top_k=20)
net.load_state_dict(synth.make_prop_state_dict())
net = net.to(dev)
eng = net.engine()
H, W, K, T, hw = 480, 864, 1, 20, 30 * 54


def timeit(fn, reps=10, warm=3):
    for _ in range(warm):
        fn()
    e0, e1 = torch.cuda.Event(True), torch.cuda.Event(True)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps, (time.perf_counter() - t0) / reps * 1e3


for N in (1, 2, 4, 8):
    frames = torch.randn(N, 3, H, W, device=dev)
    states, batch = eng.new_query_states(H, W, N)
    l0 = _lib.load().mivos_launch_count()
    g, w = timeit(lambda: net.encode_query_batch_resident(frames, batch), reps=5)
    print(f"query pass N={N}: gpu {g:.3f} ms ({g/N:.3f} ms/frame), wall {w:.3f} ms, launches/pass {(_lib.load().mivos_launch_count()-l0)//8}", flush=True)

step = FrameStep.get(net, 1, K, H, W, 30)
step.bank_k.normal_()
step.bank_v.normal_()
frame = torch.randn(1, 3, H, W, device=dev)
qs = eng.encode_query(frame)
for mem in (True, False):
    g, w = timeit(lambda: step.run([frame], [qs], T, T, mem), reps=20)
    print(f"sequential step graph (memorize={mem}): gpu {g:.3f} ms, wall {w:.3f} ms, kernels {step.kernels.get(mem)}", flush=True)
prob = torch.zeros((K + 1, 1, H, W), device=dev)


def eager():
    eng.segment(step.bank_k, step.bank_v, T * hw, qs, K, prob_out=prob)
    net.memorize_resident(frame, prob[1:], step.bank_k, step.bank_v, T)


g, w = timeit(eager, reps=10)
print(f"sequential step eager: gpu {g:.3f} ms, wall {w:.3f} ms", flush=True)
g, w = timeit(lambda: eng.segment(step.bank_k, step.bank_v, T * hw, qs, K, prob_out=prob), reps=10)
print(f"  segment only eager: gpu {g:.3f} ms, wall {w:.3f} ms", flush=True)
g, w = timeit(lambda: net.memorize_resident(frame, prob[1:], step.bank_k, step.bank_v, T), reps=10)
print(f"  memorize only eager: gpu {g:.3f} ms, wall {w:.3f} ms", flush=True)
print("done")
