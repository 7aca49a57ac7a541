"""Time every conv layer shape of the cfg-2 frame for each admissible output-channel tile width
(mivos_conv_tile_override), inside ONE process so the comparison is not confounded by box-to-box
variance.  Each (shape, BN) is captured into a CUDA graph of REPS launches and replayed, so the
number is the back-to-back launch time as it occurs inside the per-frame graph.
`python tools/tile_sweep.py residency`: the residency axis instead — every shape above and every layer of
tools/plan_table.py at n = 1, 4, 8 whose tile is narrow enough for two CTAs per SM, at the tile width and
split-K factor the planner picks, with one and with two CTAs per SM (mivos_conv_residency_override)."""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import ctypes as C
import torch
from mivos_b200 import _lib, ops

torch.set_grad_enabled(False)
dev = torch.device("cuda:0")
DT = torch.float16 if os.environ.get("MIVOS_ACT_DTYPE", "fp16") == "fp16" else torch.float32
REPS = 20

# (n, h, w, cin, cout, ks, residual)
SHAPES = [
    (1, 120, 216, 64, 256, 1, True), (1, 120, 216, 256, 64, 1, False), (1, 120, 216, 64, 64, 3, False),
    (1, 120, 216, 256, 256, 3, False), (1, 120, 216, 256, 128, 1, False),
    (1, 60, 108, 128, 512, 1, True), (1, 60, 108, 512, 128, 1, False), (1, 60, 108, 128, 128, 3, False),
    (1, 60, 108, 512, 512, 3, False), (1, 60, 108, 512, 256, 3, False), (1, 60, 108, 512, 256, 1, False),
    (1, 30, 54, 256, 1024, 1, True), (1, 30, 54, 1024, 256, 1, False), (1, 30, 54, 256, 256, 3, False),
    (1, 30, 54, 1024, 640, 3, False), (1, 30, 54, 1024, 512, 3, False), (1, 30, 54, 512, 512, 3, False),
    (8, 30, 54, 256, 1024, 1, True), (8, 30, 54, 1024, 256, 1, False), (8, 30, 54, 256, 256, 3, False),
    (8, 60, 108, 128, 512, 1, True), (8, 60, 108, 512, 128, 1, False), (8, 60, 108, 128, 128, 3, False),
    (8, 120, 216, 64, 256, 1, True), (8, 120, 216, 64, 64, 3, False),
    # the batch of a lock-step step of 4 clips (memorize trunk / decoder tail)
    (4, 120, 216, 64, 256, 1, True), (4, 60, 108, 128, 512, 1, True), (4, 30, 54, 256, 1024, 1, True),
    (4, 120, 216, 256, 256, 3, True), (4, 60, 108, 512, 256, 3, False), (4, 30, 54, 1024, 512, 3, False),
    (4, 120, 216, 256, 1, 3, False),
]
if len(sys.argv) > 1 and sys.argv[1] == "expand":  # only the output-bound 1x1 expansions
    SHAPES = [sh for sh in SHAPES if sh[5] == 1 and sh[6]]

lib = _lib.lib()


def operands(n, h, w, cin, cout, ks, res):
    wt = torch.randn(cout, cin, ks, ks, device=dev) / (cin * ks * ks) ** 0.5
    pc = ops.pack_conv(wt, torch.zeros(cout, device=dev), device=dev, dtype=DT)
    x = torch.randn((n, h + 2, w + 2, pc.cin_pad), device=dev).to(DT)
    out = torch.zeros((n, h + 2, w + 2, pc.cout_pad), device=dev, dtype=DT)
    r = torch.randn((n, h + 2, w + 2, pc.cout_pad), device=dev).to(DT) if res else None
    return pc, x, out, r


def time_us(pc, x, n, h, w, out, r):
    """us per launch of the plan the overrides currently force, in a graph of REPS back-to-back launches."""
    ops.conv_gemm(x, pc, n, h, w, out, relu=True, residual=r)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(REPS):
            ops.conv_gemm(x, pc, n, h, w, out, relu=True, residual=r)
    g.replay()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(3):
        g.replay()
    e1.record()
    torch.cuda.synchronize()
    return 1e3 * e0.elapsed_time(e1) / (3 * REPS)


def residency_sweep():
    from tools import plan_table
    shapes = list(SHAPES)
    for n in (1, 4, 8):
        for (_, h, w, cin, cout, ks, _cnt, res) in plan_table.layers():
            shapes.append((n, h, w, cin, cout, ks, res))
    print(f"dtype {DT}; us per launch (graph of {REPS} back-to-back launches) at the planned BN / split-K, "
          f"1 and 2 CTAs per SM; auto = the planner's residency")
    seen = set()
    for sh in shapes:
        if sh in seen:
            continue
        seen.add(sh)
        n, h, w, cin, cout, ks, res = sh
        pc, x, out, r = operands(*sh)
        a = ops.conv_args(x, pc, n, h, w, out, residual=r, relu=True)
        bn, sp, auto = C.c_int(0), C.c_int(0), C.c_int(0)
        _lib.check(lib.mivos_conv_plan(C.byref(a), 0, C.byref(bn), C.byref(sp)), "mivos_conv_plan")
        _lib.check(lib.mivos_conv_plan_residency(C.byref(a), 0, C.byref(auto)), "mivos_conv_plan_residency")
        if bn.value > 64:
            continue
        us = {}
        for ctas in (1, 2):
            lib.mivos_conv_residency_override(ctas)
            us[ctas] = time_us(pc, x, n, h, w, out, r)
        lib.mivos_conv_residency_override(0)
        mt = (n * (h + 2) * (w + 2) + 127) // 128
        waves = mt * (pc.cout_pad // bn.value) * sp.value / torch.cuda.get_device_properties(0).multi_processor_count
        print(f"n={n} {h:3d}x{w:3d} {cin:4d}->{cout:4d} k{ks} res={int(res)} | BN {bn.value:3d} sp {sp.value} "
              f"waves {waves:5.2f} | 1 CTA {us[1]:7.1f} | 2 CTAs {us[2]:7.1f} | 2/1 {us[2] / us[1]:5.3f} | auto {auto.value}")


if len(sys.argv) > 1 and sys.argv[1] == "residency":
    residency_sweep()
    _lib.poll_kernel_error()
    print("done")
    sys.exit(0)

print(f"dtype {DT}; us per launch (graph of {REPS} back-to-back launches); * = automatic choice")
for (n, h, w, cin, cout, ks, res) in SHAPES:
    pc, x, out, r = operands(n, h, w, cin, cout, ks, res)
    row = []
    for bn in (0, 32, 64, 128, 256):
        if bn and pc.cout_pad % bn:
            row.append("   -  ")
            continue
        lib.mivos_conv_tile_override(bn, 0)
        row.append(f"{time_us(pc, x, n, h, w, out, r):6.1f}")
    lib.mivos_conv_tile_override(0, 0)
    fl = 2.0 * n * h * w * ks * ks * cin * cout
    # least HBM traffic: the input map, the residual and the output once each (interior pixels), and the weights
    hbm = (2 if DT == torch.float16 else 4) * (n * h * w * (cin + cout * (2 if res else 1)) + ks * ks * cin * cout)
    best = min(float(v) for v in row[1:] if v.strip() != "-")
    print(f"n={n} {h:3d}x{w:3d} {cin:4d}->{cout:4d} k{ks} res={int(res)} | auto {row[0]} | 32:{row[1]} 64:{row[2]} 128:{row[3]} 256:{row[4]} | best {fl / best / 1e6:7.1f} TF/s {hbm / best / 1e3:7.1f} GB/s")
_lib.poll_kernel_error()
print("done")
