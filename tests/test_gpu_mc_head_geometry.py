"""The Monte-Carlo head (mc_exchange_kernel: default, INFO, SHARD and METRICS instantiations; and mc_combine_kernel) at
every shape and value range it accepts, against the float64 restatement tests/mc_head_ref.py.

Each case of CASES runs `world` emulated ranks on one GPU (one receive buffer, state and stream per rank), twice:
  - bbb_mc_exchange_metrics with BBB_MC_INFO over Rs sample groups x Rb row blocks: every output against
    mc_head_ref.head within mc_head_ref.bounds, epistemic >= 0 (exactly 0 for identical samples), the METRICS
    accumulator against tests/eval_ref on the returned log_outputs (bin edges as test_gpu_mc_eval counts them);
  - bbb_mc_exchange_sharded without INFO (the default or SHARD kernel): bitwise the outputs above;
  - with row blocks, bbb_mc_exchange_info on the Rs sample groups alone: bitwise the outputs above;
  - per run: NaN-prefilled outputs fully written, a sentinel guard behind each [B, C] and [B] output untouched, every
    rank bitwise identical, the second launch (other slot, next sequence number) bitwise the first; no wait timed out.
The `why` of a case names the branch it exists for; test_case_table_covers_every_branch checks the table reaches every
shape, rank count, value range and special value listed there.  Run with -s to see the worst normalised error
|got - ref| / bound per output family."""
import collections
import ctypes as C
import math
import os
import sys

import pytest
import torch

from tests import eval_ref as E
from tests import mc_head_ref as R

pytestmark = pytest.mark.gpu
# a mis-sized case fails fast on the timeout counter instead of waiting the default 10 s per word
os.environ["BBB_B200_MC_TIMEOUT_MS"] = "3000"

Case = collections.namedtuple("Case", "name why S B C world rb scale spread normalized special n_kl")


def _c(name, why, S, B, C, world=1, rb=1, scale=4.0, spread=1e-2, normalized=False, special=(), n_kl=3):
    return Case(name, why, S, B, C, world, rb, scale, spread, normalized, tuple(special), n_kl)


CASES = [
    # ---- one rank (solo: the partials never leave the registers)
    _c("solo_b1_c1", "one image, one class: p_hat = 1 in every sample", 3, 1, 1, n_kl=1),
    _c("solo_b7_c2_s7", "S_local = 7, C = 2", 7, 7, 2, scale=1.0),
    _c("solo_b8_c10_s256", "S_local = MCX_MAX_SLOCAL; samples 1e-4 apart", 256, 8, 10, spread=1e-4),
    _c("solo_b9_c31_wide", "C = 31; spread 1: samples far apart", 7, 9, 31, scale=1.0, spread=1.0),
    _c("solo_b512_c32_same", "B = 512: one row per warp; identical samples: epistemic exactly 0", 10, 512, 32, spread=0.0),
    _c("solo_b513_c33_s30", "B = 513: two rows on some warps, ragged last CTA; logit scale 30", 5, 513, 33, scale=30.0),
    _c("solo_b4099_c10_s100", "C5 per-rank work on one rank: 100 samples 1e-2 apart, B = 4099", 100, 4099, 10),
    _c("solo_b9_c10_norm_1e3", "normalized p_hat at logit scale 1e3", 4, 9, 10, scale=1e3, spread=1.0, normalized=True),
    _c("solo_b8_c1000_1e-3", "C = 1000 at logit scale 1e-3 (nearly uniform p_hat)", 6, 8, 1000, scale=1e-3, spread=1e-4),
    # ---- emulated ranks
    _c("w2_b4099_c10", "two ranks, 64 CTAs each; 13 samples per rank", 26, 4099, 10),
    _c("w3_b513_c100_norm", "three ranks with 3, 2, 2 samples; normalized; samples 1e-4 apart", 7, 513, 100, 3,
       scale=1.0, spread=1e-4, normalized=True),
    _c("w8_b512_c10_c5", "C5 over 8 ranks: 13, 13, 13, 13, 12, 12, 12, 12 samples", 100, 512, 10, 8),
    _c("w8_b9_c10_empty", "S = 3 over 8 ranks: five ranks without samples", 3, 9, 10, 8, spread=1.0),
    _c("w9_b256_c33_norm", "nine ranks: the second 8-wide batch of the finish loop", 20, 256, 33, 9, normalized=True),
    _c("w16_b256_c10", "MCX_MAX_RANKS, one sample per rank; 16 x 32 CTAs", 16, 256, 10, 16),
    _c("w16_b200_c1000", "16 ranks, C = 1000, logit scale 1e-3", 20, 200, 1000, 16, scale=1e-3, spread=1e-4),
    _c("w2_b33_c10_1e3", "logit scale 1e3: p_hat one-hot, log-probabilities far below fp32's range", 6, 33, 10, 2,
       scale=1e3, spread=1.0),
    # ---- row blocks (SHARD): world = Rs sample groups x Rb row blocks
    _c("rb2_w4_b513_c10", "Rs 2 x Rb 2, B = 513: blocks of 257 and 256 rows", 6, 513, 10, 4, 2),
    _c("rb3_w6_b7_c31", "Rs 2 x Rb 3, B = 7: blocks of 3, 2, 2", 5, 7, 31, 6, 3, spread=1.0),
    _c("rb7_w7_b7_c100", "Rs 1 x Rb = B = 7: one image per rank", 4, 7, 100, 7, 7, normalized=True),
    _c("rb2_w16_b256_c10_c5", "C5's 100 samples over Rs 8 x Rb 2", 100, 256, 10, 16, 2),
    # ---- special values
    _c("w3_b33_c10_underflow", "classes whose softmax underflows fp32 in every sample", 7, 33, 10, 3,
       special=("underflow",)),
    _c("w2_b9_c10_ties", "exact ties for the argmax: the first index wins", 4, 9, 10, 2, special=("ties",)),
    _c("w3_b9_c10_neginf", "a class at -inf in some samples but not all", 5, 9, 10, 3, special=("neginf",)),
    _c("solo_b9_c10_neginf_norm", "-inf in some samples, normalized", 5, 9, 10, normalized=True, special=("neginf",)),
    _c("w2_b9_c10_ties_norm", "ties, normalized", 4, 9, 10, 2, normalized=True, special=("ties",)),
    _c("w3_b33_c10_underflow_norm", "classes whose normalized p_hat underflows fp32 in every sample", 7, 33, 10, 3,
       normalized=True, special=("underflow",)),
]
assert len({c.name for c in CASES}) == len(CASES)


def _grid(B):
    return min(64, -(-B // 8))


def _local(S, rs, g):
    return len(range(g, S, rs))


def test_case_table_covers_every_branch():
    assert {1, 7, 8, 9, 512, 513, 4099} <= {c.B for c in CASES}
    assert {1, 2, 10, 31, 32, 33, 100, 1000} <= {c.C for c in CASES}
    sloc = {_local(c.S, c.world // c.rb, g) for c in CASES for g in range(c.world // c.rb)}
    assert {0, 1, 7, 256} <= sloc and max(sloc) == 256
    assert {c.world for c in CASES} == {1, 2, 3, 7, 8, 9, 16, 4, 6}
    assert {1, 2, 3, 8, 9, 16} <= {c.world // c.rb for c in CASES} | {c.world for c in CASES}
    shard = [c for c in CASES if c.rb > 1]
    assert any(c.B % c.rb for c in shard) and any(c.rb == c.B for c in shard)
    assert {1e-3, 1.0, 4.0, 30.0, 1e3} <= {c.scale for c in CASES}
    assert {0.0, 1e-4, 1e-2, 1.0} <= {c.spread for c in CASES}
    for sp in ("underflow", "ties", "neginf"):
        assert {False, True} == {c.normalized for c in CASES if sp in c.special}, sp
    assert any(c.n_kl > 1 for c in CASES) and any(c.n_kl == 1 for c in CASES)
    assert any(c.B > 512 and c.world > 1 for c in CASES)
    for c in CASES:                         # every rank's CTAs co-resident: 5 per SM on 132 SMs, with headroom
        assert c.world * _grid(c.B) <= 512, c.name


def _logits(cs, seed=0):
    g = torch.Generator().manual_seed(seed)
    S, B, Cc = cs.S, cs.B, cs.C
    L = cs.scale * torch.randn(1, B, Cc, generator=g) + cs.spread * torch.randn(S, B, Cc, generator=g)
    if "underflow" in cs.special:           # rows 0, 1: every class but one far below the rest in every sample
        L[:, 0, :] = torch.tensor([-200.0] * (Cc - 1) + [0.0])
        L[:, 1, : Cc // 2] = -150.0 + L[:, 1, : Cc // 2] * 1e-3
    if "ties" in cs.special:                # row 0: all classes equal; row 1: classes 3 and 7 share the maximum
        L[:, 0, :] = 0.5
        L[:, 1, :] = -1.0
        L[:, 1, 3] = L[:, 1, 7] = 2.0
        L[:, 2, :] = L[:, 2, :1]            # row 2: every class equal to the first, per sample
    if "neginf" in cs.special:              # class 2 at -inf in samples 0 and 2 of rows 0..3; class 5 in sample 1 only
        L[0, :4, 2] = -math.inf
        L[2 % S, :4, 2] = -math.inf
        L[1 % S, 1, 5] = -math.inf
    labels = torch.randint(0, Cc, (B,), generator=g)
    labels[0] = 0
    labels[-1] = Cc - 1
    if "ties" in cs.special:
        labels[1] = 3
    kl = torch.rand(cs.n_kl, generator=g) * 100.0 + 1.0
    return L.float(), labels, kl


GUARD = 64
SENT = -1.25e37
_worst = collections.defaultdict(float)


@pytest.fixture(scope="module")
def dev():
    import __graft_entry__ as g
    g.build()
    yield torch.device("cuda:0")
    if _worst:
        lines = [f"  {k:6s} worst |got - ref| / bound = {v:.3g}" for k, v in sorted(_worst.items())]
        sys.__stdout__.write("\n[mc head geometry]\n" + "\n".join(lines) + "\n")


def _buf(shape, dev):
    """An fp32 output with a sentinel guard behind it; returns (buffer, view)."""
    n = math.prod(shape)
    b = torch.full((n + GUARD,), float("nan"), dtype=torch.float32, device=dev)
    b[n:] = SENT
    return b, b[:n].view(shape)


def _run(dev, per_rank, S, B, Cc, labels, kl, normalized, info, batch_shards, entry):
    """One launch per emulated rank (`entry`: "metrics", "sharded" or "info"), twice; the outputs of every rank of the
    second launch, each checked for guards, full writes, rank equality and equality with the first launch."""
    from pytorch_bayesiancnn_b200 import _lib as L, functional as Fn, mc
    lib = L.lib()
    world = len(per_rank)
    rs = world // batch_shards
    flags = L.MC_MOMENTS | (L.MC_INFO if info else 0) | (L.MC_NORMALIZED if normalized else 0)
    nbytes = int(lib.bbb_mc_buffer_bytes(B, Cc, flags, rs))
    bufs = [torch.zeros(nbytes, dtype=torch.uint8, device=dev) for _ in range(world)]
    peers = (C.c_void_p * world)(*[b.data_ptr() for b in bufs])
    states = [torch.zeros(int(lib.bbb_mc_state_bytes()), dtype=torch.uint8, device=dev) for _ in range(world)]
    accs = [mc.new_metrics(dev) for _ in range(world)]
    streams = [torch.cuda.Stream(device=dev) for _ in range(world)]
    klt = kl.to(dev)
    lab = labels.to(dev)
    shapes = {"lo": (B, Cc), "pred": (B, Cc), "epi": (B, Cc), "ale": (B, Cc), "ent": (B,), "ee": (B,), "mi": (B,),
              "kl": (1,), "head": (4,)}
    keys = [k for k in shapes if info or k not in ("ee", "mi")]
    torch.cuda.synchronize()
    reps = []
    for rep in range(2):
        outs, raw = [], []
        for r in range(world):
            lg = per_rank[r]
            bo = {k: _buf(shapes[k], dev) for k in keys}
            o = {k: v[1] for k, v in bo.items()}
            args = (Fn._ptr(lg), 0 if lg is None else lg.shape[0], S, B, Cc, Fn._ptr(klt), klt.numel(), flags,
                    Fn._ptr(lab), C.c_float(50000.0), C.c_float(0.1), r, world, peers, Fn._ptr(states[r]),
                    Fn._ptr(o["lo"]), Fn._ptr(o["kl"]), *(Fn._ptr(o[k]) for k in ("pred", "epi", "ale", "ent", "head")),
                    None, 0, Fn._ptr(o.get("ee")), Fn._ptr(o.get("mi")))
            with torch.cuda.stream(streams[r]):
                if entry == "metrics":
                    L.check(lib.bbb_mc_exchange_metrics(*args, batch_shards, Fn._ptr(accs[r]), Fn._stream(dev)), entry)
                elif entry == "sharded":
                    L.check(lib.bbb_mc_exchange_sharded(*args, batch_shards, Fn._stream(dev)), entry)
                else:
                    L.check(lib.bbb_mc_exchange_info(*args, Fn._stream(dev)), entry)
            outs.append(o)
            raw.append(bo)
        torch.cuda.synchronize()
        for bo in raw:
            for k, (b, v) in bo.items():
                assert not torch.isnan(v).any(), (entry, k, "not fully written")
                assert bool((b[v.numel():] == SENT).all()), (entry, k, "guard overwritten")
        for o in outs[1:]:
            for k in keys:
                assert torch.equal(o[k], outs[0][k]) or _nan_equal(o[k], outs[0][k]), (entry, k, "ranks differ")
        reps.append(outs)
    for k in keys:
        assert _nan_equal(reps[0][0][k], reps[1][0][k]), (entry, k, "second launch differs")
    for st in states:
        assert int(st[8:12].view(torch.int32).item()) == 0, "an exchange wait timed out"
    if entry == "metrics":
        for a in accs[1:]:
            assert torch.equal(a[:64], accs[0][:64])
    return reps[1][0], accs[0]


def _nan_equal(a, b):
    return bool(torch.equal(a, b) or ((a == b) | (torch.isnan(a) & torch.isnan(b))).all())


def _per_rank(L, rs, rb):
    from pytorch_bayesiancnn_b200 import mc
    out = []
    for r in range(rs * rb):
        ids = list(range(r % rs, L.shape[0], rs))
        b0, b1 = mc.row_block(L.shape[1], rb, r // rs)
        out.append(L[ids][:, b0:b1].contiguous() if ids else None)
    return out


def _check(name, got, ref, bnd):
    """|got - ref| <= bnd elementwise (equal infinities allowed); the worst ratio into _worst[name]."""
    got, ref = got.double().cpu(), torch.as_tensor(ref).double()
    bnd = torch.as_tensor(bnd).double()
    same_inf = torch.isinf(ref) & (got == ref)
    err = torch.where(same_inf, torch.zeros_like(ref), (got - ref).abs())
    ratio = err / bnd.clamp_min(1e-300)
    ratio = torch.where(err == 0, torch.zeros_like(ratio), ratio)
    w = float(ratio.max()) if ratio.numel() else 0.0
    _worst[name] = max(_worst[name], w)
    if not w <= 1.0:
        i = int(torch.nan_to_num(ratio, nan=math.inf).flatten().argmax())
        raise AssertionError(f"{name}: worst |got - ref| / bound = {w:.3g} at flat index {i}: got "
                             f"{float(got.flatten()[i])!r}, ref {float(ref.flatten()[i])!r}, bound "
                             f"{float(bnd.flatten()[i]):.3g}")


@pytest.mark.parametrize("cs", CASES, ids=[c.name for c in CASES])
def test_exchange_matches_float64(dev, cs):
    from pytorch_bayesiancnn_b200 import mc
    from tests.test_gpu_mc_eval import check_against_ref
    L, labels, kl = _logits(cs)
    rs = cs.world // cs.rb
    n_loc = max(_local(cs.S, rs, g) for g in range(rs))
    n_src = rs
    per_rank = [None if t is None else t.to(dev) for t in _per_rank(L, rs, cs.rb)]
    a, acc = _run(dev, per_rank, cs.S, cs.B, cs.C, labels, kl, cs.normalized, True, cs.rb, "metrics")
    b, _ = _run(dev, per_rank, cs.S, cs.B, cs.C, labels, kl, cs.normalized, False, cs.rb, "sharded")
    for k in b:
        assert _nan_equal(a[k], b[k]), (k, "METRICS + INFO differs from the plain kernel")
    if cs.rb > 1:                          # row blocks == the sample-only exchange on the Rs sample groups
        only = [None if t is None else t.to(dev) for t in _per_rank(L, rs, 1)]
        c, _ = _run(dev, only, cs.S, cs.B, cs.C, labels, kl, cs.normalized, True, 1, "info")
        for k in c:
            assert _nan_equal(a[k], c[k]), (k, "row blocks differ from the sample-only exchange")

    ref = R.head(L, labels, kl, cs.normalized, 50000.0, 0.1)
    bnd = R.bounds(L, labels, kl, n_loc, n_src, cs.normalized, 50000.0, 0.1, ref=ref)
    assert bool((a["epi"] >= 0).all()), "negative epistemic variance"
    if cs.spread == 0.0:
        assert bool((a["epi"] == 0).all()), "identical samples: the epistemic variance is exactly 0"
    for k in ("lo", "pred", "epi", "ale", "ent", "ee", "mi"):
        _check(k, a[k], ref[k], bnd[k])
    _check("kl", a["kl"], torch.tensor([ref["kl"]]), torch.tensor([bnd["kl"]]))
    head = a["head"].double().cpu()
    _check("nll", head[1:2], torch.tensor([ref["head"][1]]), torch.tensor([bnd["nll"]]))
    _check("loss", head[0:1], torch.tensor([ref["head"][0]]), torch.tensor([bnd["loss"]]))
    _check("kl", head[3:4], torch.tensor([ref["head"][3]]), torch.tensor([bnd["beta_kl"]]))
    # accuracy: the kernel's argmax is torch.argmax of its own log_outputs (first maximal class) ...
    lo = a["lo"].cpu()
    best = lo.argmax(1)
    assert float(head[2]) == float((best == labels).double().mean().float())
    # ... and a class the float64 reference cannot tell from its maximum within the bounds
    lr, lb = ref["lo"], bnd["lo"]
    top = lr.max(1, keepdim=True).values
    ok = lr.gather(1, best[:, None])[:, 0] >= (top[:, 0] - lb.gather(1, best[:, None])[:, 0]
                                                - lb.gather(1, lr.argmax(1)[:, None])[:, 0])
    assert bool(ok.all()), "argmax outside the reference's tie band"
    if "ties" in cs.special:
        assert int(best[0]) == 0 and int(best[1]) == 3 and int(best[2]) == 0
    m = mc.read_metrics(acc)
    assert m["steps"] == 2 and m["images"] == 2 * cs.B
    s = E.batch_sums(lo, labels)
    check_against_ref(m, [s, s], cs.name)


@pytest.mark.parametrize("S,B,Cc,special", [(1, 1, 1, ()), (7, 9, 33, ()), (100, 513, 10, ()), (10000, 2, 3, ()),
                                            (5, 9, 10, ("neginf",)), (256, 8, 1000, ())])
def test_mc_combine_matches_float64(dev, S, B, Cc, special):
    """bbb_mc_combine: log_outputs within the exchange's bound (one rank); the moment planes are raw sums, against
    float64 sums within recursive-summation bounds.  S up to 10000 (40 KB of shared memory)."""
    import pytorch_bayesiancnn_b200 as bbb
    cs = _c("combine", "", S, B, Cc, spread=1e-2, special=special)
    L, _, _ = _logits(cs)
    out, mom = bbb.mc_combine(L.to(dev), want_moments=True)
    torch.cuda.synchronize()
    Ld = L.double()
    p, lp, e_p, e_lp, _ = R._per_sample(Ld, False)
    ref = O_logmeanexp(lp)
    fin = torch.isfinite(lp)
    lo_b = torch.where(fin, e_lp, torch.zeros_like(e_lp)).amax(0) + R.U * (11 * (S + 1) + 4 + 2 * math.log(S) + ref.abs())
    _check("comb_lo", out, ref, lo_b)
    ab = torch.where(torch.isfinite(Ld), Ld.abs(), torch.zeros_like(Ld))
    _check("comb_p", mom[0], p.sum(0), R.U * S * p.sum(0) + (e_p * p).sum(0))
    _check("comb_p2", mom[1], (p * p).sum(0), R.U * S * (p * p).sum(0) + (2 * e_p * p * p).sum(0))
    _check("comb_l", mom[2], Ld.sum(0), R.U * S * ab.sum(0))


def O_logmeanexp(lp):
    from oracle import bbb_oracle as O
    return O.logmeanexp(lp.permute(1, 2, 0), 2)


def test_limits_are_refused(dev):
    """S_local = MCX_MAX_SLOCAL + 1 and S = 10001 for mc_combine are refused with an error, not run."""
    import pytorch_bayesiancnn_b200 as bbb
    from pytorch_bayesiancnn_b200 import EngineError, _lib as L, functional as Fn
    lib = L.lib()
    B, Cc = 8, 10
    logits = torch.randn(257, B, Cc, device=dev)
    buf = torch.zeros(int(lib.bbb_mc_buffer_bytes(B, Cc, L.MC_MOMENTS, 1)), dtype=torch.uint8, device=dev)
    state = torch.zeros(int(lib.bbb_mc_state_bytes()), dtype=torch.uint8, device=dev)
    lo = torch.empty(B, Cc, device=dev)
    peers = (C.c_void_p * 1)(buf.data_ptr())
    rc = lib.bbb_mc_exchange_info(Fn._ptr(logits), 257, 257, B, Cc, None, 0, 0, None, C.c_float(1.0), C.c_float(0.0),
                                  0, 1, peers, Fn._ptr(state), Fn._ptr(lo), None, None, None, None, None, None, None, 0,
                                  None, None, Fn._stream(dev))
    assert rc != 0
    rc = lib.bbb_mc_exchange_info(Fn._ptr(logits), 256, 257, B, Cc, None, 0, 0, None, C.c_float(1.0), C.c_float(0.0),
                                  0, 1, peers, Fn._ptr(state), Fn._ptr(lo), None, None, None, None, None, None, None, 0,
                                  None, None, Fn._stream(dev))
    assert rc == 0
    torch.cuda.synchronize()
    bbb.mc_combine(torch.randn(10000, 1, 2, device=dev))
    with pytest.raises(EngineError):
        bbb.mc_combine(torch.randn(10001, 1, 2, device=dev))
    torch.cuda.synchronize()
