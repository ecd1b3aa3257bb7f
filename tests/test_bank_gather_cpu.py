"""The logit gather of sharded Monte-Carlo steps without a GPU: where every rank's rows land in the gathered [S, B, C]
array (the kernel's index map, and the C entry point's refusal of any other sample count), the receive-buffer size,
the rules by which a sample bank binds to a step on several ranks, and batchbald's seed on a bank of several ranks."""
import ctypes as C
import types

import pytest
import torch

LAYOUTS = [(w, rb, S, B) for w, rb, S, B in [
    (2, 1, 5, 7), (3, 1, 7, 33), (4, 2, 3, 9), (8, 2, 25, 1024), (8, 4, 3, 700), (16, 1, 100, 5), (16, 16, 1, 16),
    (16, 4, 2, 33), (3, 3, 1, 5), (6, 2, 2, 11), (8, 8, 7, 8), (4, 1, 2, 3)]]


def _placed(world, rb, S, B, Cc):
    """Each rank's local [S_local, rows, C] block of a full [S, B, C] array written at the kernel's destination index
    ((g + i Rs) B + row0) C + (b C + c), once per rank; returns the flat result and the per-word write counts."""
    from pytorch_bayesiancnn_b200 import mc
    full = torch.arange(S * B * Cc, dtype=torch.float64).view(S, B, Cc)
    out, hits = torch.full((S * B * Cc,), -1.0, dtype=torch.float64), torch.zeros(S * B * Cc, dtype=torch.int64)
    for r in range(world):
        rs, g, k = mc.shard_layout(world, r, rb)
        b0, b1 = mc.row_block(B, rb, k)
        ids = mc.local_samples(S, rs, g)
        local = full[ids][:, b0:b1].reshape(len(ids), (b1 - b0) * Cc)
        for i in range(len(ids)):
            dst0 = ((g + i * rs) * B + b0) * Cc
            out[dst0:dst0 + local.shape[1]] = local[i]
            hits[dst0:dst0 + local.shape[1]] += 1
    return full.reshape(-1), out, hits


@pytest.mark.parametrize("world,rb,S,B", LAYOUTS)
def test_every_rank_rows_land_at_their_global_position(world, rb, S, B):
    """S not a multiple of Rs, S < Rs (ranks without a sample), uneven row blocks: every word of [S, B, C] is written by
    exactly one rank, with its own value."""
    full, out, hits = _placed(world, rb, S, B, 3)
    assert torch.equal(hits, torch.ones_like(hits))
    assert torch.equal(out, full)


@pytest.mark.parametrize("world,rb,S,B", LAYOUTS)
def test_entry_point_refuses_any_other_sample_count(world, rb, S, B):
    """bbb_mc_logit_gather's argument check agrees with mc.shard_layout / local_samples on every rank: one sample more
    or one fewer than the rank's group holds is BBB_E_INVALID.  (Only refused calls here: their pointers are never
    used.  The accepted counts launch, which tests/test_gpu_bank_gather.py does with real buffers on every layout.)"""
    import __graft_entry__ as g_
    g_.build()
    from pytorch_bayesiancnn_b200 import _lib as L, mc
    lib = L.lib()
    peers = (C.c_void_p * world)(*([0x1000] * world))
    fake = C.c_void_p(0x1000)
    for r in range(world):
        rs, g, _ = mc.shard_layout(world, r, rb)
        n = len(mc.local_samples(S, rs, g))
        for s_local in (n - 1, n + 1):
            if s_local < 0:
                continue
            rc = lib.bbb_mc_logit_gather(fake, s_local, S, B, 10, r, world, rb, peers, fake, fake, None)
            assert rc == -1 and b"S_local" in lib.bbb_last_error(), (r, s_local)


def test_entry_point_refuses_bad_arguments():
    import __graft_entry__ as g_
    g_.build()
    from pytorch_bayesiancnn_b200 import _lib as L
    lib = L.lib()
    fake = C.c_void_p(0x1000)
    peers = (C.c_void_p * 4)(*([0x1000] * 4))
    ok = dict(logits=fake, S_local=1, S=4, B=8, C=10, rank=0, world=4, rb=1, peers=peers, state=fake, out=fake)

    def call(**kw):
        a = dict(ok, **kw)
        return lib.bbb_mc_logit_gather(a["logits"], a["S_local"], a["S"], a["B"], a["C"], a["rank"], a["world"],
                                       a["rb"], a["peers"], a["state"], a["out"], None)
    for kw, why in [(dict(out=None), b"NULL"), (dict(state=None), b"NULL"), (dict(peers=None), b"NULL"),
                    (dict(S=0), b"S/B/C"), (dict(B=0), b"S/B/C"), (dict(C=0), b"S/B/C"), (dict(rank=4), b"rank"),
                    (dict(world=17, rank=0), b"rank"), (dict(rank=-1), b"rank"), (dict(rb=3), b"multiple"),
                    (dict(rb=0), b"multiple"), (dict(rb=4, B=3), b"row block"), (dict(logits=None), b"NULL"),
                    (dict(peers=(C.c_void_p * 4)(0x1000, 0x1000, None, 0x1000)), b"peer buffer 2")]:
        assert call(**kw) == -1, kw
        assert why in lib.bbb_last_error(), (kw, lib.bbb_last_error())


def test_receive_buffer_bytes():
    import __graft_entry__ as g_
    g_.build()
    from pytorch_bayesiancnn_b200 import _lib as L
    lib = L.lib()
    for S, B, Cc in [(1, 1, 2), (7, 33, 10), (100, 2048, 10), (3, 700, 1000), (256, 65536, 1024)]:
        assert lib.bbb_mc_gather_bytes(S, B, Cc) == 2 * S * B * Cc * 8        # two slots of one 8-byte word per float
    assert lib.bbb_mc_gather_bytes(256, 65536, 1024) > 1 << 35             # 64-bit: past 2^31 and 2^32
    for S, B, Cc in [(0, 1, 2), (1, 0, 2), (1, 1, 0), (-1, 4, 4)]:
        assert lib.bbb_mc_gather_bytes(S, B, Cc) == 0


# --------------------------------------------------------------------------- #
# binding rules of a bank's group
# --------------------------------------------------------------------------- #
WORLD, MINE, OTHER, SOLO = (object() for _ in range(4))       # stand-ins for process groups


def _fake_dist(monkeypatch, calls=None):
    """mc._dist_info for a job of 2 ranks: SOLO has one rank, every other group two; the broadcast gives rank 0's 777."""
    from pytorch_bayesiancnn_b200 import mc

    def broadcast_object_list(box, src, group):
        calls.append((src, group))
        box[0] = 777
    dist = types.SimpleNamespace(group=types.SimpleNamespace(WORLD=WORLD), broadcast_object_list=broadcast_object_list,
                                 get_global_rank=lambda group, r: 5)
    monkeypatch.setattr(mc, "_dist_info", lambda group: (dist, 1 if group is SOLO else 2, 1))


def _step(world, group):
    return types.SimpleNamespace(world=world, group=group, dev=torch.device("cpu"), num_ens=3, C=10)


@pytest.mark.parametrize("kind", ["ProbBank", "LogitBank"])
def test_bank_binds_to_a_step_of_its_group_only(monkeypatch, kind):
    from pytorch_bayesiancnn_b200 import EngineError, mc
    _fake_dist(monkeypatch)
    make = lambda group=None: getattr(mc, kind)("cpu", 4, 3, 10, group=group)
    make(MINE)._bind(_step(2, MINE))                       # the step's group
    make(WORLD)._bind(_step(2, None))                      # a step on the default group, a bank made with it
    for group in (None, MINE, SOLO):                       # one rank: any bank, as before
        make(group)._bind(_step(1, group))
    make(MINE)._bind(_step(1, None))
    for group in (None, SOLO):                             # no group, or a group of one rank: the old refusal
        with pytest.raises(EngineError, match="needs one rank"):
            make(group)._bind(_step(2, MINE))
    with pytest.raises(EngineError, match="another group"):
        make(OTHER)._bind(_step(2, MINE))
    with pytest.raises(EngineError, match="another group"):
        make(MINE)._bind(_step(2, None))
    with pytest.raises(EngineError, match=f"{make()._keyword} holds"):
        getattr(mc, kind)("cpu", 4, 4, 10, group=MINE)._bind(_step(2, MINE))
    e = make(MINE)._empty()                                # what the warm-up steps append to
    assert e.group is MINE and e.capacity == 0
    e._bind(_step(2, MINE))


def test_batchbald_seed_is_rank0s_on_a_bank_of_several_ranks(monkeypatch):
    from pytorch_bayesiancnn_b200 import mc
    calls = []
    _fake_dist(monkeypatch, calls)
    bank = lambda group: mc.ProbBank("cpu", 4, 3, 10, group=group)
    assert mc._selection_seed(bank(MINE), None) == 777 and calls == [(5, MINE)]
    calls.clear()
    assert mc._selection_seed(bank(MINE), 12) == 12 and calls == []         # a given seed is every rank's already
    drawn = mc._selection_seed(bank(None), None)                          # no group: this rank's own draw
    assert drawn != 777 and 0 <= drawn < 1 << 62 and calls == []
    assert mc._selection_seed(bank(SOLO), None) != 777 and calls == []     # a group of one rank: nothing to share


def test_step_seed_is_still_rank0s(monkeypatch):
    """MCForward's seed goes through the same broadcast (the default group when group=None, src 0)."""
    from pytorch_bayesiancnn_b200 import mc
    calls = []
    _fake_dist(monkeypatch, calls)
    assert mc._from_rank0(3, None) == 777 and calls == [(0, None)]
    assert mc._from_rank0(3, MINE) == 777 and calls[-1] == (5, MINE)
    assert mc._from_rank0(3, SOLO) == 3 and len(calls) == 2
