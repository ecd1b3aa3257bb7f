"""Float64 reference of the information outputs of the Monte-Carlo step (helpers, not a test module).

The entropy decomposition of the MC predictive distribution, per image:
    H[p_bar]  =  E_s H[p_hat_s]  +  I(y; w)
    (entropy)    (expected entropy)  (mutual information)
with p_hat_s = softmax(logits_s), or softplus(logits_s) / sum softplus with ``normalized``
(uncertainty_estimation.py:73-77), and H[p] = -sum_c p_c log p_c, 0 log 0 = 0.
"""
from typing import Sequence

import torch
import torch.nn.functional as F


def p_hat(logits_per_sample: Sequence[torch.Tensor], normalized=False) -> torch.Tensor:
    """[T, B, C] float64 per-sample class probabilities, as oracle.bbb_oracle.uncertainty forms them."""
    L = torch.stack([torch.as_tensor(l) for l in logits_per_sample], 0).double()
    if normalized:
        pr = F.softplus(L)
        return pr / pr.sum(2, keepdim=True)
    return F.softmax(L, dim=2)


def _entropy(p: torch.Tensor) -> torch.Tensor:
    """-sum over the last dim of p log p, with 0 log 0 = 0."""
    return -torch.where(p > 0, p * torch.log(torch.where(p > 0, p, torch.ones_like(p))), torch.zeros_like(p)).sum(-1)


def information(logits_per_sample: Sequence[torch.Tensor], normalized=False):
    """(expected_entropy [B], mutual_info [B]) in float64: mean_s H[p_hat_s] and H[p_bar] - mean_s H[p_hat_s]."""
    p = p_hat(logits_per_sample, normalized)
    expected = _entropy(p).mean(0)
    return expected, _entropy(p.mean(0)) - expected
