"""Float64 restatement of main_bayesian.validate_model (main_bayesian.py:65-86, metrics.py) and of the calibration
figures of the evaluation accumulator (include/bbb_b200.h, bbb_mc_exchange_metrics), vectorised over a batch.

Per image, on p_bar = exp(log_outputs): conf = p_bar[argmax] (first maximal class), correct = argmax == y,
nll = -log_outputs[y], brier = sum_c (p_bar_c - [c == y])^2, calibration bin m = clamp(ceil(15 conf) - 1, 0, 14)."""
import math

import torch

BINS = 15


def bin_of(conf):
    """Calibration bin of each confidence (float64 tensor): the equal-width bins (m/15, (m+1)/15]."""
    return (torch.ceil(conf * BINS) - 1).clamp(0, BINS - 1).long()


def batch_sums(log_outputs, labels):
    """The accumulator's per-image sums of one batch, in float64: nll, correct, brier and, per bin, count / conf /
    correct; also the per-image conf for the bin-edge accounting of the tests."""
    lo = torch.as_tensor(log_outputs).double()
    y = torch.as_tensor(labels).long()
    p = lo.exp()
    best = lo.argmax(1)                                   # first maximal class, like the kernel
    conf = p.gather(1, best[:, None])[:, 0]
    correct = (best == y).double()
    nll = -lo.gather(1, y[:, None])[:, 0]
    onehot = torch.zeros_like(p).scatter_(1, y[:, None], 1.0)
    brier = ((p - onehot) ** 2).sum(1)
    m = bin_of(conf)
    z = torch.zeros(BINS, dtype=torch.float64)
    return {"images": lo.shape[0], "nll": float(nll.sum()), "correct": float(correct.sum()), "brier": float(brier.sum()),
            "bin_count": z.clone().index_add_(0, m, torch.ones_like(conf)),
            "bin_conf": z.clone().index_add_(0, m, conf), "bin_correct": z.clone().index_add_(0, m, correct),
            "conf": conf}


def summarize(sums):
    """What read_metrics reports from the summed batch sums (a list of batch_sums results)."""
    n = sum(s["images"] for s in sums)
    cnt = sum(s["bin_count"] for s in sums)
    conf = sum(s["bin_conf"] for s in sums)
    cor = sum(s["bin_correct"] for s in sums)
    nan = float("nan")
    return {"images": n, "nll": sum(s["nll"] for s in sums) / n, "accuracy": sum(s["correct"] for s in sums) / n,
            "brier": sum(s["brier"] for s in sums) / n, "ece": float((cor - conf).abs().sum()) / n,
            "bin_count": [int(c) for c in cnt],
            "bin_confidence": [float(conf[m] / cnt[m]) if cnt[m] else nan for m in range(BINS)],
            "bin_accuracy": [float(cor[m] / cnt[m]) if cnt[m] else nan for m in range(BINS)]}


def get_beta(batch_idx, m, beta_type, epoch=None, num_epochs=None):
    """metrics.py:32-46."""
    if type(beta_type) is float:
        return beta_type
    if beta_type == "Blundell":
        return 2 ** (m - (batch_idx + 1)) / (2 ** m - 1)
    if beta_type == "Soenderby":
        return min(epoch / (num_epochs // 4), 1)
    if beta_type == "Standard":
        return 1 / m
    return 0


def validate(log_outputs, labels, klsums, train_size, beta_type=0.1, epoch=None, num_epochs=None):
    """validate_model's (valid_loss, valid_acc) from each batch's log_outputs, labels and kl = sum_j kl_j."""
    n = len(log_outputs)
    loss, accs = 0.0, []
    for i, (lo, y, kl) in enumerate(zip(log_outputs, labels, klsums)):
        lo, y = torch.as_tensor(lo).double(), torch.as_tensor(y).long()
        beta = get_beta(i - 1, n, beta_type, epoch, num_epochs)
        nll = float(-lo.gather(1, y[:, None]).mean())
        loss += nll * train_size + beta * float(kl)
        accs.append(float((lo.argmax(1) == y).double().mean()))
    return loss / n, sum(accs) / n


def per_image_loop(log_outputs, labels):
    """The same sums one image and one class at a time (plain Python floats): the check on batch_sums."""
    out = {"nll": 0.0, "correct": 0.0, "brier": 0.0, "bin_count": [0.0] * BINS, "bin_conf": [0.0] * BINS,
           "bin_correct": [0.0] * BINS}
    for row, y in zip(torch.as_tensor(log_outputs).double().tolist(), torch.as_tensor(labels).tolist()):
        p = [math.exp(v) for v in row]
        best = max(range(len(row)), key=lambda c: (row[c], -c))
        conf, hit = p[best], 1.0 if best == y else 0.0
        out["nll"] -= row[y]
        out["correct"] += hit
        out["brier"] += sum((p[c] - (1.0 if c == y else 0.0)) ** 2 for c in range(len(p)))
        m = min(max(math.ceil(conf * BINS) - 1, 0), BINS - 1)
        out["bin_count"][m] += 1
        out["bin_conf"][m] += conf
        out["bin_correct"][m] += hit
    return out
