"""Eager fused-chain forwards of BBBAlexNet (B=512) for ncu captures:
    ncu --set full --import-source on -k regex:conv_s4_kernel -s 2 -c 1 -o prof python tools/ncu_fwd.py [lrt|bbb] [reps]"""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import pytorch_bayesiancnn_b200 as bbb
from bench import build_net
variant = sys.argv[1] if len(sys.argv) > 1 else "lrt"
reps = int(sys.argv[2]) if len(sys.argv) > 2 else 4
dev = torch.device("cuda:0")
net = build_net(variant, 10, dev, "bf16")
xs = [torch.randn(512, 3, 32, 32, device=dev) for _ in range(reps)]
bbb.manual_seed(1)
with torch.no_grad():
    for x in xs:
        out, kl = net(x)
torch.cuda.synchronize()
print("ok", float(kl))
