"""CPU-only: the tile width / split-K plan `mivos_conv_gemm` picks (mivos_conv_plan, pure host arithmetic)
for every convolution of the sequential step (segment + memorize) at cfg-2, for a batch of n = C*K maps —
n = 1 is one clip, n = 4 a lock-step lane of four.  Prints row tiles, CTAs, waves on the SMs and the
tensor work per launch, to see which layers the batch lifts over one wave and which it does not.
Usage: python tools/plan_table.py [--sms S=132 (H100 SXM)] [n ...=1 4 8]"""
import ctypes as C
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from mivos_b200 import _lib  # noqa: E402

SMS = 132  # H100 SXM
H, W = 480, 864


def layers():
    """(name, h, w, cin, cout, ksize, count per frame, residual, im2col) of the sequential step."""
    out = []
    h4, w4, h8, w8, h16, w16 = H // 4, W // 4, H // 8, W // 8, H // 16, W // 16
    # memorize trunk (mask_rgb_encoder): stem + layer1..3 + kv projection
    out.append(("stem 7x7/2 5->64 (im2col K=256)", H // 2, W // 2, 256, 64, 1, 1, False))
    for name, (h, w), planes, blocks, cin in (("layer1", (h4, w4), 64, 3, 64), ("layer2", (h8, w8), 128, 4, 256),
                                              ("layer3", (h16, w16), 256, 6, 512)):
        out.append((f"{name} 1x1 {cin}->{planes} (block 0)", h if name == "layer1" else 2 * h, w if name == "layer1" else 2 * w, cin, planes, 1, 1, False))
        out.append((f"{name} 1x1 {4 * planes}->{planes}", h, w, 4 * planes, planes, 1, blocks - 1, False))
        if name == "layer1":
            out.append((f"{name} 3x3 {planes}->{planes}", h, w, planes, planes, 3, blocks, False))
        else:
            out.append((f"{name} 3x3/2 {planes}->{planes} (im2col)", h, w, 9 * planes, planes, 1, 1, False))
            out.append((f"{name} 3x3 {planes}->{planes}", h, w, planes, planes, 3, blocks - 1, False))
        out.append((f"{name} 1x1 {planes}->{4 * planes} +res", h, w, planes, 4 * planes, 1, blocks, True))
        out.append((f"{name} downsample 1x1 {cin}->{4 * planes}", h, w, cin, 4 * planes, 1, 1, False))
    out.append(("kv_m 3x3 1024->640", h16, w16, 1024, 640, 3, 1, False))
    # decoder tail
    out.append(("compress conv1 3x3 1024->512", h16, w16, 1024, 512, 3, 1, False))
    out.append(("compress downsample 3x3 1024->512", h16, w16, 1024, 512, 3, 1, False))
    out.append(("compress conv2 3x3 512->512 +res", h16, w16, 512, 512, 3, 1, True))
    out.append(("up_16_8 out conv1 3x3 512->256", h8, w8, 512, 256, 3, 1, False))
    out.append(("up_16_8 out downsample 3x3 512->256", h8, w8, 512, 256, 3, 1, False))
    out.append(("up_16_8 out conv2 3x3 256->256 +res", h8, w8, 256, 256, 3, 1, True))
    out.append(("up_8_4 out conv1/conv2 3x3 256->256", h4, w4, 256, 256, 3, 2, True))
    out.append(("pred 3x3 256->1", h4, w4, 256, 1, 3, 1, False))
    return out


def plan(n, h, w, cin, cout, ks, residual, sms=SMS):
    a = _lib.ConvArgs()
    a.n, a.h, a.w = n, h, w
    a.cin_pad = (cin + 63) // 64 * 64
    a.taps = 9 if ks == 3 else 1
    a.cout, a.cout_pad = cout, (cout + 31) // 32 * 32
    a.in_f16 = a.out_f16 = 1
    a.residual = 1 if residual else 0
    a.splitk_ws, a.splitk_ws_bytes = 1, 48 << 20
    bn, sp = C.c_int(0), C.c_int(0)
    assert _lib.load().mivos_conv_plan(C.byref(a), sms, C.byref(bn), C.byref(sp)) == 0
    rows = n * (h + 2) * (w + 2)
    mt = (rows + 127) // 128
    ctas = mt * (a.cout_pad // bn.value) * sp.value
    return bn.value, sp.value, mt, ctas


def main():
    args, sms = sys.argv[1:], SMS
    if args[:1] == ["--sms"]:
        sms, args = int(args[1]), args[2:]
    ns = [int(x) for x in args] or [1, 4, 8]
    print(f"{'layer':44s} {'x':>2s} " + " ".join(f"| n={n}: BN sp tiles CTAs waves  GF" for n in ns))
    tot = {n: 0.0 for n in ns}
    for name, h, w, cin, cout, ks, cnt, res in layers():
        cells = []
        for n in ns:
            bn, sp, mt, ctas = plan(n, h, w, cin, cout, ks, res, sms)
            gf = 2.0 * n * h * w * cin * cout * (9 if ks == 3 else 1) / 1e9
            cells.append(f"| {bn:8d} {sp:2d} {mt:5d} {ctas:4d} {ctas / sms:5.2f} {gf:5.1f}")
            tot[n] += ctas / sms * cnt
        print(f"{name:44s} {cnt:2d} " + " ".join(cells))
    print(f"sum of (CTAs/{sms}) x count per frame-step: " + ", ".join(f"n={n}: {tot[n]:.1f} ({tot[n] / n:.1f} per clip)" for n in ns))


if __name__ == "__main__":
    main()
