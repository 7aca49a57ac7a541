"""Time every conv layer shape of the cfg-2 frame for each admissible output-channel tile width
(mivos_conv_tile_override), inside ONE process so the comparison is not confounded by box-to-box
variance.  Each (shape, BN) is captured into a CUDA graph of REPS launches and replayed, so the
number is the back-to-back launch time as it occurs inside the per-frame graph."""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
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
print(f"dtype {DT}; us per launch (graph of {REPS} back-to-back launches); * = automatic choice")
for (n, h, w, cin, cout, ks, res) in SHAPES:
    wt = torch.randn(cout, cin, ks, ks, device=dev) / (cin * ks * ks) ** 0.5
    pc = ops.pack_conv(wt, torch.zeros(cout, device=dev), device=dev, dtype=DT)
    x = torch.randn((n, h + 2, w + 2, pc.cin_pad), device=dev).to(DT)
    out = torch.zeros((n, h + 2, w + 2, pc.cout_pad), device=dev, dtype=DT)
    r = torch.randn((n, h + 2, w + 2, pc.cout_pad), device=dev).to(DT) if res else None
    row = []
    for bn in (0, 32, 64, 128, 256):
        if bn and pc.cout_pad % bn:
            row.append("   -  ")
            continue
        lib.mivos_conv_tile_override(bn, 0)
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
        row.append(f"{1e3 * e0.elapsed_time(e1) / (3 * REPS):6.1f}")
    lib.mivos_conv_tile_override(0, 0)
    fl = 2.0 * n * h * w * ks * ks * cin * cout
    best = min(float(v) for v in row[1:] if v.strip() != "-")
    print(f"n={n} {h:3d}x{w:3d} {cin:4d}->{cout:4d} k{ks} res={int(res)} | auto {row[0]} | 32:{row[1]} 64:{row[2]} 128:{row[3]} 256:{row[4]} | best {fl / best / 1e6:7.1f} TF/s")
_lib.poll_kernel_error()
print("done")
