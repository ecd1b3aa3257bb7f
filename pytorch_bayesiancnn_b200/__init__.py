"""H100-native Bayes-by-Backprop layer engine (hot path of kumar-shridhar/PyTorch-BayesianCNN).

Public surface = the reference's ``layers`` exports (layers/__init__.py:1-7) plus the
engine controls.  The compute lives in libbbb_b200.so (csrc/, C ABI in include/bbb_b200.h).
"""
from .modules import (BBBConv2d, BBBLinear, BBBLRTConv2d, BBBLRTLinear, FlattenLayer, ModuleWrapper, posterior_as_prior,
                      mixture_prior, snr, prune_by_snr)
from .functional import (manual_seed, begin_sample, external_eps, philox_normal, mc_combine)
from .graph import GraphedForward
from . import functional
from ._lib import EngineError, launch_count, LIB_PATH

BBB_Linear = BBBLinear
BBB_Conv2d = BBBConv2d
BBB_LRT_Linear = BBBLRTLinear
BBB_LRT_Conv2d = BBBLRTConv2d

__all__ = ["BBB_Linear", "BBB_Conv2d", "BBB_LRT_Linear", "BBB_LRT_Conv2d", "FlattenLayer", "ModuleWrapper",
           "BBBConv2d", "BBBLinear", "BBBLRTConv2d", "BBBLRTLinear", "manual_seed", "begin_sample",
           "external_eps", "philox_normal", "mc_combine", "EngineError", "launch_count", "LIB_PATH",
           "posterior_as_prior", "mixture_prior", "snr", "prune_by_snr"]
