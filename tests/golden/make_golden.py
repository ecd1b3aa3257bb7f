"""Generate golden fixtures by running the UNMODIFIED reference on the CPU.

    PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_golden.py /path/to/PyTorch-BayesianCNN

Imports the original project (read-only) -- never copied into the repo -- runs its
layers / models on seeded inputs, recovers the eps it drew by seed-replay of the
global CPU generator (SURVEY.md 8c), and writes small ``.npz`` files next to
this script.  The suite never needs the original project, so nothing in the
test-suite calls this script; it is committed so the fixtures are reproducible.

Fixtures
  layers.npz  : per-layer cases (x, params, eps, y, kl) for conv/linear x bbb/lrt
  models.npz  : the three model files, both variants: x, logits, kl, and float64
                checksums of every parameter (params are re-drawn from the seed
                by oracle.init_params; the checksums prove the re-draw matches)
"""
import os
import sys

sys.dont_write_bytecode = True
REF = sys.argv[1] if len(sys.argv) > 1 else "."
HERE = os.path.dirname(os.path.abspath(__file__))
# the reference's layer files do `sys.path.append("..")` and import top-level
# `metrics`; run with the reference root first on sys.path, like `cd reference`.
sys.path.insert(0, REF)
os.chdir(REF)

import numpy as np
import torch

import layers as ref_layers                      # noqa: E402  (the reference's)
from models.BayesianModels.BayesianAlexNet import BBBAlexNet        # noqa: E402
from models.BayesianModels.BayesianLeNet import BBBLeNet            # noqa: E402
from models.BayesianModels.Bayesian3Conv3FC import BBB3Conv3FC      # noqa: E402
import config_bayesian as cfg                   # noqa: E402

torch.set_num_threads(1)        # oneDNN single-thread: deterministic reduction order

DEFAULT_PRIORS = None           # layer default: rho ~ N(-3, 0.1)
CFG_PRIORS = cfg.priors         # config_bayesian.py:4-9: rho ~ N(-5, 0.1)

# name, kind, variant, ctor args, ctor kwargs, x shape, priors, x distribution
LAYER_CASES = [
    ("conv_bbb_k3",      "conv", "bbb", (3, 8, 3),   dict(stride=1, padding=1),            (2, 3, 8, 8),   DEFAULT_PRIORS, "randn"),
    ("conv_bbb_k5s2",    "conv", "bbb", (4, 6, 5),   dict(stride=2, padding=2),            (3, 4, 11, 9),  CFG_PRIORS,     "rand"),
    ("conv_bbb_dil",     "conv", "bbb", (2, 5, 3),   dict(stride=1, padding=2, dilation=2), (2, 2, 9, 9),  DEFAULT_PRIORS, "randn"),
    ("conv_bbb_nobias",  "conv", "bbb", (3, 4, 3),   dict(padding=0, bias=False),          (2, 3, 6, 6),   DEFAULT_PRIORS, "randn"),
    ("conv_bbb_rect",    "conv", "bbb", (3, 4, (3, 5)), dict(padding=1),                   (2, 3, 7, 9),   DEFAULT_PRIORS, "randn"),
    ("conv_bbb_alex1",   "conv", "bbb", (3, 64, 11), dict(stride=4, padding=5),            (2, 3, 32, 32), CFG_PRIORS,     "rand"),
    ("conv_lrt_k3",      "conv", "lrt", (3, 8, 3),   dict(stride=1, padding=1),            (2, 3, 8, 8),   DEFAULT_PRIORS, "randn"),
    ("conv_lrt_k5s2",    "conv", "lrt", (4, 6, 5),   dict(stride=2, padding=2),            (3, 4, 11, 9),  CFG_PRIORS,     "rand"),
    ("conv_lrt_dil",     "conv", "lrt", (2, 5, 3),   dict(stride=1, padding=2, dilation=2), (2, 2, 9, 9),  DEFAULT_PRIORS, "randn"),
    ("conv_lrt_nobias",  "conv", "lrt", (3, 4, 3),   dict(padding=0, bias=False),          (2, 3, 6, 6),   DEFAULT_PRIORS, "randn"),
    ("conv_lrt_alex1",   "conv", "lrt", (3, 64, 11), dict(stride=4, padding=5),            (2, 3, 32, 32), CFG_PRIORS,     "rand"),
    ("conv_lrt_alex3",   "conv", "lrt", (48, 96, 3), dict(padding=1),                      (2, 48, 2, 2), CFG_PRIORS,     "rand"),
    ("lin_bbb_small",    "lin",  "bbb", (7, 5),      dict(),                               (3, 7),         DEFAULT_PRIORS, "randn"),
    ("lin_bbb_cls",      "lin",  "bbb", (128, 10),   dict(),                               (16, 128),      CFG_PRIORS,     "rand"),
    ("lin_bbb_nobias",   "lin",  "bbb", (33, 17),    dict(bias=False),                     (5, 33),        DEFAULT_PRIORS, "randn"),
    ("lin_lrt_small",    "lin",  "lrt", (7, 5),      dict(),                               (3, 7),         DEFAULT_PRIORS, "randn"),
    ("lin_lrt_cls",      "lin",  "lrt", (128, 10),   dict(),                               (16, 128),      CFG_PRIORS,     "rand"),
    ("lin_lrt_fc",       "lin",  "lrt", (400, 120),  dict(),                               (4, 400),       CFG_PRIORS,     "randn"),
    ("lin_lrt_nobias",   "lin",  "lrt", (33, 17),    dict(bias=False),                     (5, 33),        DEFAULT_PRIORS, "randn"),
]

MODEL_CASES = [
    # name, class, arch key, inputs, outputs, variant, act, batch
    ("alexnet_bbb",  BBBAlexNet,  "alexnet",  3, 10,  "bbb", "softplus", 4),
    ("alexnet_lrt",  BBBAlexNet,  "alexnet",  3, 10,  "lrt", "softplus", 4),
    ("alexnet100_lrt", BBBAlexNet, "alexnet", 3, 100, "lrt", "relu",     2),
    ("lenet_bbb",    BBBLeNet,    "lenet",    3, 10,  "bbb", "softplus", 4),
    ("lenet_lrt",    BBBLeNet,    "lenet",    3, 10,  "lrt", "relu",     4),
    ("3conv3fc_bbb", BBB3Conv3FC, "3conv3fc", 1, 10,  "bbb", "softplus", 3),
    ("3conv3fc_lrt", BBB3Conv3FC, "3conv3fc", 1, 10,  "lrt", "softplus", 3),
]
PARAM_SEED, X_SEED, EPS_SEED = 123, 0, 7


def make_x(shape, dist, seed):
    g = torch.Generator().manual_seed(seed)
    if dist == "rand":
        return torch.rand(shape, generator=g)
    return torch.randn(shape, generator=g)


def layer_case(name, kind, variant, args, kwargs, xshape, priors, dist, out):
    mods = {("conv", "bbb"): ref_layers.BBB_Conv2d, ("conv", "lrt"): ref_layers.BBB_LRT_Conv2d,
            ("lin", "bbb"): ref_layers.BBB_Linear, ("lin", "lrt"): ref_layers.BBB_LRT_Linear}
    torch.manual_seed(PARAM_SEED)
    layer = mods[(kind, variant)](*args, priors=priors, **kwargs)
    layer.train()
    x = make_x(xshape, dist, X_SEED)
    with torch.no_grad():
        torch.manual_seed(EPS_SEED)
        y = layer(x)
        kl = layer.kl_loss()
        # seed-replay: re-issue the same draws (BBB/BBBConv.py:63,68; BBB_LRT/BBBConv.py:78)
        torch.manual_seed(EPS_SEED)
        if variant == "bbb":
            eps_w = torch.empty(layer.W_mu.size()).normal_(0, 1)
            eps_b = torch.empty(layer.bias_mu.size()).normal_(0, 1) if layer.use_bias else None
        else:
            eps_y = torch.empty(y.size()).normal_(0, 1)
        # deterministic (mean-only) path: forward(x, sample=False) in eval mode
        layer.eval()
        y_mean = layer(x, sample=False)
    pre = name + "/"
    out[pre + "x"] = x.numpy()
    out[pre + "W_mu"] = layer.W_mu.detach().numpy()
    out[pre + "W_rho"] = layer.W_rho.detach().numpy()
    if layer.use_bias:
        out[pre + "bias_mu"] = layer.bias_mu.detach().numpy()
        out[pre + "bias_rho"] = layer.bias_rho.detach().numpy()
    if variant == "bbb":
        out[pre + "eps_w"] = eps_w.numpy()
        if eps_b is not None:
            out[pre + "eps_b"] = eps_b.numpy()
    else:
        out[pre + "eps_y"] = eps_y.numpy()
    out[pre + "y"] = y.numpy()
    out[pre + "y_mean"] = y_mean.numpy()
    out[pre + "kl"] = np.float32(kl.item())
    out[pre + "prior"] = np.array([layer.prior_mu, layer.prior_sigma], np.float64)
    if kind == "conv":
        def pair(v):
            return list(v) if isinstance(v, tuple) else [v, v]
        out[pre + "conv"] = np.array(pair(layer.stride) + pair(layer.padding) + pair(layer.dilation), np.int64)


def model_case(name, cls, key, inputs, outputs, variant, act, batch, out):
    torch.manual_seed(PARAM_SEED)
    net = cls(outputs, inputs, CFG_PRIORS, variant, act)
    net.train()
    x = make_x((batch, inputs, 32, 32), "randn", X_SEED)
    with torch.no_grad():
        torch.manual_seed(EPS_SEED)
        logits, kl = net(x)
    pre = name + "/"
    out[pre + "x"] = x.numpy()
    out[pre + "logits"] = logits.numpy()
    out[pre + "kl"] = np.float32(float(kl))
    out[pre + "meta"] = np.array([key, str(inputs), str(outputs), variant, act, str(batch)])
    sums = [float(p.detach().double().sum()) for _, p in net.named_parameters()]
    out[pre + "param_sums"] = np.array(sums, np.float64)
    out[pre + "param_names"] = np.array([n for n, _ in net.named_parameters()])


def main():
    lay = {}
    for c in LAYER_CASES:
        layer_case(*c, lay)
    np.savez_compressed(os.path.join(HERE, "layers.npz"), **lay)
    mod = {}
    for c in MODEL_CASES:
        model_case(*c, mod)
    np.savez_compressed(os.path.join(HERE, "models.npz"), **mod)
    print("layers.npz", os.path.getsize(os.path.join(HERE, "layers.npz")),
          "models.npz", os.path.getsize(os.path.join(HERE, "models.npz")))
    print("torch", torch.__version__)


if __name__ == "__main__":
    main()
