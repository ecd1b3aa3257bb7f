"""A small run of every wgmma / mbarrier / TMA kernel for compute-sanitizer (racecheck, synccheck, memcheck) -- the
empty/full barrier rings and the accumulators staged over the operand ring and the staged images:
    compute-sanitizer --tool racecheck python tools/sanitize_fwd.py
BBBAlexNet, batch 48 (ragged tiles), LRT and BBB, fused chain (conv_s4 + tap-GEMMs) + the MC exchange kernel, no graphs."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import pytorch_bayesiancnn_b200 as bbb
from pytorch_bayesiancnn_b200 import mc
from bench import build_net
dev = torch.device("cuda:0")
for variant in ("lrt", "bbb"):
    net = build_net(variant, 10, dev, "bf16")
    x = torch.randn(48, 3, 32, 32, device=dev)
    eng = mc.MCForward(net, x, 2, want_uncertainty=True, seed=3, graph=False)
    out = eng(x)
    torch.cuda.synchronize()
    assert torch.isfinite(out["log_outputs"]).all()
    layer = net.conv2                                  # the generic gather kernel too (unfused layer call)
    with torch.no_grad():
        y = layer(torch.randn(8, 64, 4, 4, device=dev))
    torch.cuda.synchronize()
    layer.set_flag("math", "tf32")                     # and its tf32-operand instance
    with torch.no_grad():
        y = layer(torch.randn(8, 64, 4, 4, device=dev))
    layer.set_flag("math", "bf16")
    torch.cuda.synchronize()
    print(variant, "ok", float(out["kl"]), tuple(y.shape))
