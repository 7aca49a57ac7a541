"""Where does the wall time of one cfg-2 interact() go?  CPU time per phase of the frame loop and
GPU time (CUDA events on the main stream around each frame step, on the side stream around each
batched query pass).  No profiler: perf_counter + events only."""
import sys, os, time, collections
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import mivos_b200
from mivos_b200 import synth
from mivos_b200.frame_step import FrameStep

torch.set_grad_enabled(False)
dev = torch.device("cuda:0")
net = mivos_b200.PropagationNetwork(top_k=20)
net.load_state_dict(synth.make_prop_state_dict())
net = net.to(dev)
T = int(os.environ.get("FRAMES", "101"))
images, mask = synth.synthetic_clip(T, 480, 854, 1, seed=1234)


CORES = [mivos_b200.InferenceCore(net, None, images, 1, mem_profile=0, mem_freq=5, device=dev) for _ in range(6)]


def one(instrument):
    core = CORES.pop()
    cpu = collections.defaultdict(float)
    ev = {"step": [], "chunk": []}
    if instrument:
        orig_run, orig_get, orig_issue = FrameStep.run, core.get_query_kv_buffered, core._issue_query_chunk

        def run(self, *a, **k):
            t0 = time.perf_counter()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            r = orig_run(self, *a, **k)
            e1.record()
            ev["step"].append((e0, e1))
            cpu["step.run"] += time.perf_counter() - t0
            return r

        def get(*a, **k):
            t0 = time.perf_counter()
            r = orig_get(*a, **k)
            cpu["get_query"] += time.perf_counter() - t0
            return r

        def issue(want):
            t0 = time.perf_counter()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            core._qstream.wait_stream(torch.cuda.current_stream())
            e0.record(core._qstream)
            r = orig_issue(want)
            e1.record(core._qstream)
            ev["chunk"].append((e0, e1, len(want)))
            cpu["issue_chunk"] += time.perf_counter() - t0
            return r

        FrameStep.run = run
        core.get_query_kv_buffered = get
        core._issue_query_chunk = issue
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0 = time.perf_counter()
    a.record()
    m = core.interact(mask, 0)
    b.record()
    t_issue = time.perf_counter() - t0
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0
    if instrument:
        FrameStep.run = orig_run
    return wall, t_issue, a.elapsed_time(b), cpu, ev


for _ in range(2):
    one(False)
wall, t_issue, gpu, _, _ = one(False)
print(f"plain:        wall {wall*1e3:.1f} ms, python returns after {t_issue*1e3:.1f} ms, events {gpu:.1f} ms  ({(T-1)/wall:.1f} fps)")
wall, t_issue, gpu, cpu, ev = one(True)
print(f"instrumented: wall {wall*1e3:.1f} ms, python returns after {t_issue*1e3:.1f} ms, events {gpu:.1f} ms")
for k, v in cpu.items():
    print(f"  cpu {k:12s} {v*1e3:8.1f} ms total")
st = [a.elapsed_time(b) for a, b in ev["step"]]
print(f"  main-stream frame steps: n={len(st)} sum {sum(st):.1f} ms, mean {sum(st)/len(st):.3f}, min {min(st):.3f}, max {max(st):.3f}")
ck = [(a.elapsed_time(b), n) for a, b, n in ev["chunk"]]
print(f"  side-stream query chunks: n={len(ck)} sum {sum(c for c, _ in ck):.1f} ms; per chunk " + " ".join(f"{c:.2f}/{n}" for c, n in ck))
gaps = [ev["step"][i][1].elapsed_time(ev["step"][i + 1][0]) for i in range(len(st) - 1)]
print(f"  gaps between frame steps on the main stream: sum {sum(gaps):.1f} ms, max {max(gaps):.3f}")
print("  first 24 step durations:", " ".join(f"{x:.2f}" for x in st[:24]))
print("  first 24 gaps:", " ".join(f"{x:.2f}" for x in gaps[:24]))
import cProfile, pstats, io
core = CORES.pop()
torch.cuda.synchronize()
pr = cProfile.Profile()
pr.enable()
core.interact(mask, 0)
pr.disable()
buf = io.StringIO()
pstats.Stats(pr, stream=buf).sort_stats("tottime").print_stats(16)
print(buf.getvalue()[:6000])
print("done")
