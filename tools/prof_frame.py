"""One steady-state cfg-2 frame (query encoder -> memory read -> decoder -> aggregate -> memorize)
repeated a few times; run under `ncu --metrics gpu__time_duration.sum` for the per-kernel launch list."""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import mivos_b200
from mivos_b200 import synth

torch.set_grad_enabled(False)
dev = torch.device("cuda:0")
net = mivos_b200.PropagationNetwork(top_k=20)
net.load_state_dict(synth.make_prop_state_dict())
net = net.to(dev)
K, T, hw = 1, 20, 30 * 54
frame = torch.randn(1, 3, 480, 864, device=dev)
bank_k = torch.randn((K, (T + 1) * hw, 128), device=dev)
bank_v = torch.randn((K, (T + 1) * hw, 512), device=dev)
reps = int(sys.argv[1]) if len(sys.argv) > 1 else 3
qs = None
for i in range(reps):
    torch.cuda.nvtx.range_push("frame")
    qs = net.encode_query_resident(frame, qs)
    _, prob = net.engine().segment(bank_k, bank_v, T * hw, qs, K)
    net.memorize_resident(frame, prob[1:], bank_k, bank_v, T)
    torch.cuda.nvtx.range_pop()
torch.cuda.synchronize()
print("done")
