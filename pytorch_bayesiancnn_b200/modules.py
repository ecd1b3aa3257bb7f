"""The reference's layer surface (SURVEY.md 8b) on top of the CUDA engine.

Same class names, constructor signatures, parameter names (``W_mu``, ``W_rho``,
``bias_mu``, ``bias_rho`` -- the state_dict keys), ``forward(x, sample=True)``,
``kl_loss()``, ``reset_parameters()``, ``ModuleWrapper.set_flag`` and
``FlattenLayer`` as layers/BBB/BBBConv.py, layers/BBB/BBBLinear.py,
layers/BBB_LRT/BBBConv.py, layers/BBB_LRT/BBBLinear.py and layers/misc.py, so that
models/BayesianModels/*.py import and train unchanged.  The bodies are new: one
fused CUDA kernel per forward (through the C ABI), KL computed in that kernel.

Engine knobs ride on ``set_flag`` (never on the constructor):
  math           'fp32' | 'bf16' | 'tf32' | 'auto'   arithmetic path (default from $BBB_B200_MATH or 'auto': the tensor-core
                                            path wherever the shape fits a wgmma tile, IEEE-fp32 CUDA cores otherwise;
                                            'fp32' forces the exact-arithmetic kernels everywhere)
  kl_convention  'reference' | 'textbook'   default 'reference' = the formula as executed (SURVEY D1)

Per-weight Gaussian priors (``set_prior`` / ``posterior_as_prior``): the KL of every parameter element is taken against
its own N(mu_p, sigma_p^2), e.g. the posterior of a previous task (variational continual learning) or a prior centred on
pretrained weights.  The prior lives in four fp32 buffers (``W_prior_mu``, ``W_prior_sigma``, ``bias_prior_mu``,
``bias_prior_sigma``) that exist only after ``set_prior``: a layer that never had one keeps the reference's state_dict.

Scale-mixture priors (``set_mixture_prior`` / ``mixture_prior``): the prior Bayes by Backprop was published with (Blundell
et al. 2015, section 3.3), pi N(0, sigma1^2) + (1 - pi) N(0, sigma2^2).  It has no closed-form KL: the layer's KL is then
a Monte-Carlo estimate of KL(q || p) from one weight draw per layer call (functional.KLMCFn), on a Philox stream of the
call's own, so every Monte-Carlo sample has its own estimate.  ``kl_convention`` does not apply to it.  A layer has one
prior: the scalar pair, the tensors or the mixture.  The mixture's three values live in the fp32 buffer
``mixture_prior``, which exists only after ``set_mixture_prior``.

Pruning (``set_weight_mask`` / ``prune_by_snr``): a bool mask per layer removes weights (and optionally biases) from the
model.  A pruned element is a deterministic zero in every forward, adds nothing to the KL and gets exactly zero gradient
on every path of the engine; kept elements compute exactly what they compute without a mask.  The mask lives in the bool
buffers ``W_mask`` / ``bias_mask``, which exist only after ``set_weight_mask``.  A pruned net is not faster: the kernels
still multiply the zeros.
"""
from __future__ import annotations

import math
import os

import torch
from torch import nn
from torch.nn import Parameter

from . import _lib as L
from . import functional as Fn

_DEFAULT_PRIORS = {
    "prior_mu": 0,
    "prior_sigma": 0.1,
    "posterior_mu_initial": (0, 0.1),
    "posterior_rho_initial": (-3, 0.1),
}
_PRIOR_BUFFERS = ("W_prior_mu", "W_prior_sigma", "bias_prior_mu", "bias_prior_sigma")
_MIXTURE_BUFFER = "mixture_prior"
_MASK_BUFFERS = ("W_mask", "bias_mask")
_prior_epoch = 0          # bumped whenever some layer's prior buffers are created, replaced, moved or removed (PriorGuard)


def _prior_moved():
    global _prior_epoch
    _prior_epoch += 1


def _default_math() -> str:
    return os.environ.get("BBB_B200_MATH", "auto")


def _default_fuse() -> bool:
    return os.environ.get("BBB_B200_FUSE", "1") != "0"


class ModuleWrapper(nn.Module):
    """layers/misc.py:4-25: universal forward returning (x, kl); recursive set_flag."""

    def __init__(self):
        super().__init__()

    def set_flag(self, flag_name, value):
        setattr(self, flag_name, value)
        self.__dict__.pop("_fused_plans", None)          # engine knobs (math, fuse, ...) change what can be fused
        for child in self.children():
            if hasattr(child, "set_flag"):
                child.set_flag(flag_name, value)

    def _try_fused(self, x):
        """Run the children as a fused tensor-core chain if they match (see fused.py); None = not fusable."""
        if not (torch.is_tensor(x) and x.is_cuda and x.dim() == 4) or not getattr(self, "fuse", _default_fuse()):
            return None
        if Fn.layer_fold_active():
            return None                                    # MC samples folded on the per-layer path (Fn.layer_fold)
        if torch.is_grad_enabled() and (x.requires_grad or any(p.requires_grad for p in self.parameters())):
            return None                                    # the fused chain is forward-only
        from . import fused
        plans = self.__dict__.setdefault("_fused_plans", {})
        key = tuple(x.shape)
        if key not in plans:
            kids = list(self.children())
            plans[key] = fused.plan(kids, tuple(x.shape)) if kids else None
        steps = plans[key]
        if steps is None:
            return None
        try:
            return fused.run(steps, x)          # (output, summed KL)
        except L.EngineError as e:
            if "code -2" not in str(e):                    # anything but BBB_E_UNSUPPORTED is a real error
                raise
            plans[key] = None
            return None

    def forward(self, x):
        out = self._try_fused(x)
        if out is not None:
            # the fused chain already reduced the per-layer KL scalars (each layer's kl_loss() still
            # returns its own term); same value as the loop below, one launch instead of one per layer
            if x.dtype == torch.bfloat16:                  # the chain upcasts a bf16 input once: bf16 in, bf16 out
                return out[0].to(torch.bfloat16), out[1]
            return out
        for child in self.children():
            x = child(x)
        kl = 0.0
        for m in self.modules():
            if hasattr(m, "kl_loss"):
                kl = kl + m.kl_loss()
        return x, kl


class FlattenLayer(ModuleWrapper):
    """layers/misc.py:28-35: x.view(-1, num_features) (no shape check, like the reference)."""

    def __init__(self, num_features):
        super().__init__()
        self.num_features = num_features

    def forward(self, x):
        return x.reshape(-1, self.num_features) if not x.is_contiguous() else x.view(-1, self.num_features)


def _pair(v):
    return tuple(v) if isinstance(v, (tuple, list)) else (v, v)


class _BayesLayer(ModuleWrapper):
    """Shared machinery of the four reference layer classes."""
    _variant = L.VARIANT_BBB
    _params_on_device = True       # BBB creates params on cuda:0 if present (BBB/BBBConv.py:27,41);
                                   # LRT on CPU (BBB_LRT/BBBConv.py:43-44) -- kept (SURVEY D12)

    def _setup(self, w_shape, n_out, bias, priors):
        self.use_bias = bias
        self.device = torch.device("cuda:0" if torch.cuda.is_available() else "cpu")
        if priors is None:
            priors = dict(_DEFAULT_PRIORS)
        self.prior_mu = priors["prior_mu"]
        self.prior_sigma = priors["prior_sigma"]
        self.posterior_mu_initial = priors["posterior_mu_initial"]
        self.posterior_rho_initial = priors["posterior_rho_initial"]
        dev = self.device if self._params_on_device else torch.device("cpu")
        self.W_mu = Parameter(torch.empty(w_shape, device=dev))
        self.W_rho = Parameter(torch.empty(w_shape, device=dev))
        if self.use_bias:
            self.bias_mu = Parameter(torch.empty(n_out, device=dev))
            self.bias_rho = Parameter(torch.empty(n_out, device=dev))
        else:
            self.register_parameter("bias_mu", None)
            self.register_parameter("bias_rho", None)
        self.math = _default_math()
        self.kl_convention = "reference"
        self._kl_cache = None
        self._mixture = None           # (pi, sigma1, sigma2) after set_mixture_prior: the host's copy of the buffer
        self.reset_parameters()

    def reset_parameters(self):
        self.W_mu.data.normal_(*self.posterior_mu_initial)
        self.W_rho.data.normal_(*self.posterior_rho_initial)
        if self.use_bias:
            self.bias_mu.data.normal_(*self.posterior_mu_initial)
            self.bias_rho.data.normal_(*self.posterior_rho_initial)

    # -- engine plumbing ------------------------------------------------------
    def _conv_geometry(self):
        return None

    def _versions(self):
        """What a cached KL scalar depends on: the parameters' versions AND the KL settings (changing
        kl_convention or the prior -- scalar or tensor (set_prior) -- after a forward must not return the old value)."""
        ps = (self.W_mu, self.W_rho, self.bias_mu, self.bias_rho) + tuple(
            self._buffers.get(n) for n in _PRIOR_BUFFERS + _MASK_BUFFERS)
        return tuple((p._version, p.data_ptr()) if p is not None else None for p in ps) + (
            self.kl_convention, float(self.prior_mu), float(self.prior_sigma), self.mixture_values())

    # -- per-weight priors ----------------------------------------------------
    def prior_tensors(self):
        """(W_prior_mu, W_prior_sigma, bias_prior_mu, bias_prior_sigma) after set_prior (bias ones None without a
        bias), or None: the KL is taken against the scalar prior_mu / prior_sigma."""
        if self._buffers.get("W_prior_mu") is None:
            return None
        return tuple(self._buffers.get(n) for n in _PRIOR_BUFFERS)

    def set_prior(self, mu=None, sigma=None, bias_mu=None, bias_sigma=None):
        """Take the KL against a per-element Gaussian prior N(mu, sigma^2) from now on.  Each argument is a number or a
        tensor that broadcasts to the shape of W_mu (mu, sigma) or bias_mu (bias_mu, bias_sigma); None takes the layer's
        scalar prior_mu / prior_sigma.  The values are stored as contiguous fp32 buffers on the parameters' device, so
        they follow .to() / .cuda() and are saved in the state_dict.  sigma must be finite and > 0 (ValueError; checked
        here, not by the kernels).  Setting again with the same shapes copies in place: the buffers keep their
        addresses, so an engine captured after the first set_prior (MCForward, GraphedForward) reads the new values on
        its next replay.  No gradient flows to the prior."""
        if not self.use_bias and (bias_mu is not None or bias_sigma is not None):
            raise ValueError("set_prior: the layer has no bias")
        dev = self.W_mu.device
        parts = [("W_prior_mu", mu, self.prior_mu, self.W_mu.shape, False),
                 ("W_prior_sigma", sigma, self.prior_sigma, self.W_mu.shape, True)]
        if self.use_bias:
            parts += [("bias_prior_mu", bias_mu, self.prior_mu, self.bias_mu.shape, False),
                      ("bias_prior_sigma", bias_sigma, self.prior_sigma, self.bias_mu.shape, True)]
        vals = []
        for name, v, scalar, shape, is_sigma in parts:
            t = torch.as_tensor(scalar if v is None else v).detach().to(device=dev, dtype=torch.float32)
            try:
                ok = torch.broadcast_shapes(t.shape, shape) == shape
            except RuntimeError:
                ok = False
            if not ok:
                raise ValueError(f"set_prior: {name} of shape {tuple(t.shape)} does not broadcast to {tuple(shape)}")
            if not bool(torch.isfinite(t).all()) or (is_sigma and not bool((t > 0).all())):
                raise ValueError(f"set_prior: {name} must be finite" + (" and > 0" if is_sigma else ""))
            vals.append((name, t, shape))
        for name, t, shape in vals:
            buf = self._buffers.get(name)
            if buf is not None and buf.shape == shape and buf.device == dev and buf.is_contiguous():
                with torch.no_grad():
                    buf.copy_(t)
            else:
                self.register_buffer(name, torch.empty(shape, dtype=torch.float32, device=dev).copy_(t))
                _prior_moved()
        self._drop_mixture()
        return self

    # -- pruning mask ---------------------------------------------------------
    def mask_tensors(self):
        """(W_mask, bias_mask) after set_weight_mask (bias_mask None when every bias is kept), or None: no mask."""
        if self._buffers.get("W_mask") is None:
            return None
        return self._buffers.get("W_mask"), self._buffers.get("bias_mask")

    def set_weight_mask(self, W_mask, bias_mask=None):
        """Prune the layer: from now on a weight whose W_mask element is False (a bias, with ``bias_mask``; without one
        every bias is kept) is a deterministic zero in the forward, adds nothing to the KL and gets exactly zero gradient
        in mu and rho, on every path of the engine.  The kept elements are computed exactly as without a mask (same noise,
        same bits).  Masks are bool tensors of exactly the shape of W_mu / bias_mu on the parameters' device (ValueError
        otherwise); they are stored in the buffers ``W_mask`` / ``bias_mask``, follow .to() and are saved in the
        state_dict.  Setting again with the same shapes copies in place: an engine captured after the first
        set_weight_mask (MCForward, GraphedForward) reads the new mask on its next replay.  Not with a mixture prior
        (ValueError): its Monte-Carlo KL takes no mask."""
        if self.mixture_values() is not None:
            raise ValueError("set_weight_mask: the layer has a mixture prior, whose Monte-Carlo KL takes no mask")
        if bias_mask is not None and not self.use_bias:
            raise ValueError("set_weight_mask: the layer has no bias")
        parts = [("W_mask", W_mask, self.W_mu)]
        if bias_mask is not None:
            parts.append(("bias_mask", bias_mask, self.bias_mu))
        for name, t, like in parts:
            if not torch.is_tensor(t) or t.dtype != torch.bool:
                raise ValueError(f"set_weight_mask: {name} must be a torch.bool tensor, got "
                                 f"{t.dtype if torch.is_tensor(t) else type(t).__name__}")
            if t.shape != like.shape:
                raise ValueError(f"set_weight_mask: {name} of shape {tuple(t.shape)}, expected {tuple(like.shape)}")
            if t.device != like.device:
                raise ValueError(f"set_weight_mask: {name} is on device {t.device}, the parameters on {like.device}")
        for name, t, like in parts:
            buf = self._buffers.get(name)
            if buf is not None and buf.shape == like.shape and buf.device == like.device and buf.is_contiguous():
                with torch.no_grad():
                    buf.copy_(t)
            else:
                self.register_buffer(name, t.detach().clone(memory_format=torch.contiguous_format))
                _prior_moved()
        if bias_mask is None and self._buffers.pop("bias_mask", None) is not None:
            _prior_moved()
        return self

    def clear_weight_mask(self):
        """Keep every element again: removes the mask buffers.  A captured engine that read them refuses its next replay
        (PriorGuard); mc_forward / evaluate build new engines."""
        removed = [self._buffers.pop(n, None) for n in _MASK_BUFFERS]
        if any(t is not None for t in removed):
            _prior_moved()
        return self

    # -- scale-mixture prior --------------------------------------------------
    def mixture_values(self):
        """(pi, sigma1, sigma2) after set_mixture_prior, or None: the prior is a Gaussian (scalar or tensor)."""
        return self.__dict__.get("_mixture")

    def set_mixture_prior(self, pi=0.5, sigma1=1.0, sigma2=math.exp(-6)):
        """Take the KL against the scale mixture pi N(0, sigma1^2) + (1 - pi) N(0, sigma2^2) from now on (Blundell et al.
        2015, section 3.3; usually sigma1 > sigma2, a wide slab and a narrow spike).  The layer's KL becomes a Monte-Carlo
        estimate of KL(q || p): every layer call draws one weight sample for it on a Philox stream id of its own, taken
        after the layer's noise stream (the layer's outputs do not change), and under an MC-sample fold one per sample.
        kl_convention does not apply.  0 < pi <= 1 and finite sigma1, sigma2 > 0 (ValueError).  Replaces a tensor prior
        (set_prior); clear_prior goes back to the scalar prior.  The values are kept, rounded to fp32, in the 3-element
        buffer ``mixture_prior`` -- saved in the state_dict, following .to() -- and passed to the kernels by value: a
        captured engine (MCForward, GraphedForward) refuses its next replay once they changed (PriorGuard); mc_forward
        and evaluate build new engines.  Change them through this method, not by writing to the buffer."""
        vals = _check_mixture(pi, sigma1, sigma2)
        if self.mask_tensors() is not None:
            raise ValueError("set_mixture_prior: the layer has a weight mask; the mixture prior's Monte-Carlo KL takes "
                             "no mask (clear_weight_mask first)")
        self.clear_prior()
        self.register_buffer(_MIXTURE_BUFFER, torch.tensor(vals, dtype=torch.float32, device=self.W_mu.device))
        self._mixture = vals
        _prior_moved()
        return self

    def _drop_mixture(self):
        if self._buffers.pop(_MIXTURE_BUFFER, None) is not None or self.mixture_values() is not None:
            self._mixture = None
            _prior_moved()

    def clear_prior(self):
        """Back to the scalar prior_mu / prior_sigma: removes the prior buffers.  A captured engine that read them
        refuses its next replay (PriorGuard); mc_forward / evaluate build new engines."""
        removed = [self._buffers.pop(n, None) for n in _PRIOR_BUFFERS]
        if any(t is not None for t in removed):
            _prior_moved()
        self._drop_mixture()
        return self

    def _apply(self, fn, *args, **kwargs):
        # .to() / .cuda() / .float() replace the buffers: engines captured on the old ones must notice
        out = super()._apply(fn, *args, **kwargs)
        if self._buffers.get("W_prior_mu") is not None or self._buffers.get("W_mask") is not None:
            _prior_moved()
        return out

    def _load_from_state_dict(self, state_dict, prefix, local_metadata, strict, missing_keys, unexpected_keys,
                              error_msgs):
        # a checkpoint saved after set_prior carries the prior: create the buffers so that it loads into a fresh layer.
        # They take the parameters' shapes, so a checkpoint prior of another shape fails torch's size check.
        shapes = {"W_prior_mu": self.W_mu.shape, "W_prior_sigma": self.W_mu.shape}
        if self.use_bias:
            shapes.update(bias_prior_mu=self.bias_mu.shape, bias_prior_sigma=self.bias_mu.shape)
        for n, shape in shapes.items():
            if prefix + n in state_dict and self._buffers.get(n) is None:
                self.register_buffer(n, torch.zeros(shape, dtype=torch.float32, device=self.W_mu.device))
                _prior_moved()
        # likewise a pruning mask (bool, the parameters' shapes)
        masks = {"W_mask": self.W_mu.shape}
        if self.use_bias:
            masks["bias_mask"] = self.bias_mu.shape
        for n, shape in masks.items():
            if prefix + n in state_dict and self._buffers.get(n) is None:
                self.register_buffer(n, torch.ones(shape, dtype=torch.bool, device=self.W_mu.device))
                _prior_moved()
        # likewise the mixture prior; its values are read back to the host once, here
        has_mix = prefix + _MIXTURE_BUFFER in state_dict
        if has_mix and self._buffers.get(_MIXTURE_BUFFER) is None:
            self.register_buffer(_MIXTURE_BUFFER, torch.zeros(3, dtype=torch.float32, device=self.W_mu.device))
        super()._load_from_state_dict(state_dict, prefix, local_metadata, strict, missing_keys, unexpected_keys,
                                      error_msgs)
        if has_mix and tuple(self._buffers[_MIXTURE_BUFFER].shape) == (3,):
            try:
                self._mixture = _check_mixture(*self._buffers[_MIXTURE_BUFFER].tolist())
            except ValueError as e:
                error_msgs.append(f"{prefix}{_MIXTURE_BUFFER}: {e}")
                self._buffers.pop(_MIXTURE_BUFFER)
                self._mixture = None
            _prior_moved()

    def _cfg(self, sample):
        return {
            "conv": self._conv_geometry(),
            "variant": self._variant,
            "sample": bool(sample),
            "prior_mu": float(self.prior_mu),
            "prior_sigma": float(self.prior_sigma),
            "math": L.MATH_BY_NAME[self.math],
            "kl_convention": L.KL_BY_NAME[self.kl_convention],
            "act": L.ACT_NONE,
            "owner": self,
            "prior": self.prior_tensors(),
            "mixture": self.mixture_values(),
            "mask": self.mask_tensors(),
        }

    def forward(self, x, sample=True):
        stochastic = bool(self.training or sample)      # BBB/BBBConv.py:62, BBB_LRT/BBBConv.py:77
        cfg = self._cfg(stochastic)
        cfg["grad_enabled"] = torch.is_grad_enabled()  # grad mode is always off inside Function.forward
        y, kl = Fn.BayesLayerFn.apply(x, self.W_mu, self.W_rho, self.bias_mu, self.bias_rho, cfg)
        if cfg["mixture"] is not None:                  # the forward computed no KL: one Monte-Carlo draw per MC sample
            kl = Fn.KLMCFn.apply(self.W_mu, self.W_rho, self.bias_mu, self.bias_rho, cfg["mixture"],
                                 Fn.fold_draws(x.shape[0]), self)
        self._kl_cache = (kl, self._versions(), torch.is_grad_enabled())
        return y

    def kl_loss(self):
        """0-dim tensor, differentiable w.r.t. mu and rho.  Normally the scalar the
        fused forward kernel just produced; recomputed by the stand-alone KL kernel
        if no forward preceded it or the parameters changed since (the reference
        would raise AttributeError / use a stale sigma there -- SURVEY D7).  With a mixture prior the scalar is a
        Monte-Carlo estimate: the preceding forward's draw (under an MC-sample fold, one per sample: a vector), or a new
        draw on the next Philox stream id when there is none."""
        c = self._kl_cache
        if c is not None and c[1] == self._versions() and (c[2] or not torch.is_grad_enabled()):
            return c[0]
        if self.mixture_values() is not None:
            return Fn.KLMCFn.apply(self.W_mu, self.W_rho, self.bias_mu, self.bias_rho, self.mixture_values(), None, self)
        return Fn.KLFn.apply(self.W_mu, self.W_rho, self.bias_mu, self.bias_rho, float(self.prior_mu),
                             float(self.prior_sigma), L.KL_BY_NAME[self.kl_convention], self.prior_tensors(),
                             self.mask_tensors())

    @property
    def W_sigma(self):
        """The reference caches log1p(exp(W_rho)) as a forward side effect
        (BBB/BBBConv.py:64); kept as a read-only view for code that inspects it."""
        return torch.log1p(torch.exp(self.W_rho))

    @W_sigma.setter
    def W_sigma(self, value):
        pass                                             # the reference assigns it in forward; derived here

    @property
    def bias_sigma(self):
        return torch.log1p(torch.exp(self.bias_rho)) if self.use_bias else None

    @bias_sigma.setter
    def bias_sigma(self, value):
        pass


class _ConvMixin:
    def _init_conv(self, in_channels, out_channels, kernel_size, stride, padding, dilation, bias, priors):
        self.in_channels = in_channels
        self.out_channels = out_channels
        self.kernel_size = _pair(kernel_size)
        self.stride = stride
        self.padding = padding
        self.dilation = dilation
        self.groups = 1
        self._setup((out_channels, in_channels, *self.kernel_size), out_channels, bias, priors)

    def _conv_geometry(self):
        return (_pair(self.stride), _pair(self.padding), _pair(self.dilation))


class BBBConv2d(_ConvMixin, _BayesLayer):
    """layers/BBB/BBBConv.py:14 -- weight-space sampling conv."""
    _variant = L.VARIANT_BBB

    def __init__(self, in_channels, out_channels, kernel_size,
                 stride=1, padding=0, dilation=1, bias=True, priors=None):
        super().__init__()
        self._init_conv(in_channels, out_channels, kernel_size, stride, padding, dilation, bias, priors)


class BBBLRTConv2d(_ConvMixin, _BayesLayer):
    """layers/BBB_LRT/BBBConv.py:16 -- local-reparameterisation conv."""
    _variant = L.VARIANT_LRT
    _params_on_device = False

    def __init__(self, in_channels, out_channels, kernel_size, stride=1,
                 padding=0, dilation=1, bias=True, priors=None):
        super().__init__()
        self._init_conv(in_channels, out_channels, kernel_size, stride, padding, dilation, bias, priors)


class _LinearMixin:
    def _init_linear(self, in_features, out_features, bias, priors):
        self.in_features = in_features
        self.out_features = out_features
        self._setup((out_features, in_features), out_features, bias, priors)


class BBBLinear(_LinearMixin, _BayesLayer):
    """layers/BBB/BBBLinear.py:14."""
    _variant = L.VARIANT_BBB

    def __init__(self, in_features, out_features, bias=True, priors=None):
        super().__init__()
        self._init_linear(in_features, out_features, bias, priors)


class BBBLRTLinear(_LinearMixin, _BayesLayer):
    """layers/BBB_LRT/BBBLinear.py:16."""
    _variant = L.VARIANT_LRT
    _params_on_device = False

    def __init__(self, in_features, out_features, bias=True, priors=None):
        super().__init__()
        self._init_linear(in_features, out_features, bias, priors)


def _check_mixture(pi, sigma1, sigma2):
    """(pi, sigma1, sigma2) rounded to fp32, as the engine takes them; ValueError unless 0 < pi <= 1 and sigma1, sigma2
    are finite, > 0 and have squares within fp32 range (what bbb_kl_mc_forward checks)."""
    pi, sigma1, sigma2 = torch.tensor([float(pi), float(sigma1), float(sigma2)], dtype=torch.float32).tolist()
    if not 0.0 < pi <= 1.0:
        raise ValueError(f"mixture prior: pi must be in (0, 1], got {pi}")
    for name, v in (("sigma1", sigma1), ("sigma2", sigma2)):
        if not (math.isfinite(v) and v > 0.0):
            raise ValueError(f"mixture prior: {name} must be finite and > 0, got {v}")
        h = torch.tensor(0.5 / (v * v), dtype=torch.float32).item()
        if not math.isfinite(h) or h == 0.0:
            raise ValueError(f"mixture prior: {name}^2 is outside fp32 range, got {v}")
    return pi, sigma1, sigma2


def has_mixture(net: nn.Module) -> bool:
    """Does a Bayesian layer of `net` take its KL against a mixture prior (a per-sample Monte-Carlo estimate)?"""
    return any(isinstance(m, _BayesLayer) and m.mixture_values() is not None for m in net.modules())


def prior_signature(net: nn.Module) -> tuple:
    """What a captured graph holds of every Bayesian layer's prior: the tensor prior's buffer addresses, the mixture
    prior's values (kernel arguments), or None for the scalar prior."""
    def one(m):
        if m.mixture_values() is not None:
            return ("mixture",) + m.mixture_values()
        if m.prior_tensors() is None:
            return None
        return tuple(None if t is None else t.data_ptr() for t in m.prior_tensors())
    return tuple(one(m) for m in net.modules() if isinstance(m, _BayesLayer))


def mask_signature(net: nn.Module) -> tuple:
    """What a captured graph holds of every Bayesian layer's weight mask: the mask buffers' addresses, or None."""
    def one(m):
        ts = m.mask_tensors()
        return None if ts is None else tuple(None if t is None else t.data_ptr() for t in ts)
    return tuple(one(m) for m in net.modules() if isinstance(m, _BayesLayer))


class PriorGuard:
    """The layers' priors and weight masks as a captured CUDA graph of `net` bakes them in: the buffers' addresses, or
    NULL for a scalar prior / no mask.  It holds the buffers, so a replay never reads freed memory, and ``ok()`` tells whether a replay still reads
    what the layers hold: false once a prior was set for the first time, cleared, re-allocated or moved.  An in-place
    set_prior keeps the addresses (the next replay reads the new values).  While no layer anywhere changed its prior's
    identity, ``ok()`` is one integer compare."""

    def __init__(self, net: nn.Module):
        self.net, self.epoch, self.sig = net, _prior_epoch, (prior_signature(net), mask_signature(net))
        self.keep = [t for m in net.modules() if isinstance(m, _BayesLayer)
                     for t in (m.prior_tensors() or ()) + (m.mask_tensors() or ()) if t is not None]

    def ok(self) -> bool:
        if self.epoch == _prior_epoch:
            return True
        if (prior_signature(self.net), mask_signature(self.net)) != self.sig:
            return False
        self.epoch = _prior_epoch
        return True

    def check(self, what: str):
        if not self.ok():
            raise L.EngineError(f"{what}: a layer's prior or weight mask was set, cleared, re-allocated or moved since this "
                                "engine's CUDA graphs were captured; build a new engine (an in-place set_prior or "
                                "set_weight_mask of the same shapes is read by the next replay; new set_mixture_prior "
                                "values are not)")


def posterior_as_prior(net: nn.Module) -> nn.Module:
    """The continual-learning step (variational continual learning, Nguyen et al. 2018): every Bayesian layer of `net`
    takes its current posterior N(W_mu, softplus(W_rho)^2), element by element, as the prior of its KL from now on
    (set_prior; the bias likewise).  Train task A, call this, then train task B: the KL pulls the weights towards what
    task A learned, in proportion to how certain it was.  sigma = log1p(exp(rho)), the engine's softplus."""
    for m in net.modules():
        if isinstance(m, _BayesLayer):
            with torch.no_grad():
                m.set_prior(m.W_mu.detach(), torch.log1p(torch.exp(m.W_rho.detach())),
                            m.bias_mu.detach() if m.use_bias else None,
                            torch.log1p(torch.exp(m.bias_rho.detach())) if m.use_bias else None)
    return net


def mixture_prior(net: nn.Module, pi=0.5, sigma1=1.0, sigma2=math.exp(-6)) -> nn.Module:
    """Give every Bayesian layer of `net` the scale-mixture prior pi N(0, sigma1^2) + (1 - pi) N(0, sigma2^2) of Blundell
    et al. 2015 (set_mixture_prior): the net's KL is from then on the sum of the layers' Monte-Carlo estimates, one draw
    per layer and Monte-Carlo sample."""
    for m in net.modules():
        if isinstance(m, _BayesLayer):
            m.set_mixture_prior(pi, sigma1, sigma2)
    return net


def snr(layer: _BayesLayer) -> torch.Tensor:
    """Signal-to-noise ratio of every weight of a Bayesian layer, |W_mu| / sigma with sigma = log1p(exp(W_rho)) in fp32
    as the reference computes it (Blundell et al. 2015, section 5.1): the shape of W_mu, on its device."""
    return _snr(layer.W_mu, layer.W_rho)


def _snr(mu, rho):
    mu, rho = mu.detach().float(), rho.detach().float()
    return mu.abs() / torch.log1p(torch.exp(rho))


def prune_by_snr(net: nn.Module, fraction: float, biases: bool = False) -> dict:
    """Prune the weights of every Bayesian layer of `net` with the lowest signal-to-noise ratio (snr), as Blundell et al.
    2015 (section 5.1) do: one ranking over all layers' weights (and biases, with ``biases``), of which exactly
    floor(fraction * N) are pruned, lowest SNR first, ties broken by (layer order in net.modules(), flat index).
    Elements a layer's mask already prunes rank first, so ``fraction`` is the share pruned in total, and pruning again
    never brings an element back (a fraction below the share already pruned leaves the masks as they are).  The masks
    are set with set_weight_mask (without ``biases`` a layer's bias mask is left as it was).  Runs on the parameters'
    device with torch ops.  Returns {"pruned", "total", "threshold" (the SNR of the last element pruned by this call;
    None when it prunes nothing), "per_layer": {name: (pruned, total)}}."""
    fraction = float(fraction)
    if not 0.0 <= fraction <= 1.0:
        raise ValueError(f"prune_by_snr: fraction must be in [0, 1], got {fraction}")
    layers = [(name, m) for name, m in net.named_modules() if isinstance(m, _BayesLayer)]
    keys, sizes = [], []
    for _, m in layers:
        parts = [(m.W_mu, m.W_rho, 0)] + ([(m.bias_mu, m.bias_rho, 1)] if biases and m.use_bias else [])
        masks = m.mask_tensors() or (None, None)
        for mu, rho, j in parts:
            k = _snr(mu, rho).reshape(-1)
            if masks[j] is not None:
                k = k.masked_fill(~masks[j].reshape(-1), -math.inf)
            keys.append(k)
            sizes.append(k.numel())
    if not keys:
        return {"pruned": 0, "total": 0, "threshold": None, "per_layer": {}}
    dev = keys[0].device
    key = torch.cat([k.to(dev) for k in keys])
    total = key.numel()
    already = int((key == -math.inf).sum())
    n = max(int(math.floor(fraction * total)), already)
    order = torch.sort(key, stable=True).indices
    pruned = torch.zeros(total, dtype=torch.bool, device=dev)
    pruned[order[:n]] = True
    threshold = None
    if n > already:
        threshold = float(key[order[n - 1]])
    per_layer, off, it = {}, 0, iter(sizes)
    for name, m in layers:
        ranked = [m.W_mu] + ([m.bias_mu] if biases and m.use_bias else [])
        cut = []
        for t in ranked:
            sz = next(it)
            cut.append(pruned[off:off + sz].view(t.shape).to(t.device))
            off += sz
        bias_keep = ~cut[1] if len(cut) > 1 else (m.mask_tensors() or (None, None))[1]
        m.set_weight_mask(~cut[0], bias_keep)
        per_layer[name] = (int(sum(int(c.sum()) for c in cut)), sum(c.numel() for c in cut))
    return {"pruned": n, "total": total, "threshold": threshold, "per_layer": per_layer}
