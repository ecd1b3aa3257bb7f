"""Row-block sharding of the Monte-Carlo step without a GPU: the (sample group, row block) partition, the first-image
field of the layer desc, the host-only support queries, and the generic path over gloo with batch_shards 1, 2, 4."""
import ctypes
import os
import socket
import tempfile

import pytest
import torch
import torch.multiprocessing as mp

from tests.util import CFG_PRIORS


@pytest.fixture(scope="module")
def built():
    import __graft_entry__ as g
    g.build()
    return g.LIB


@pytest.mark.parametrize("world", [1, 2, 3, 4, 8])
def test_partition_covers_every_sample_row_pair_once(world):
    from pytorch_bayesiancnn_b200 import mc
    for rb in [d for d in range(1, world + 1) if world % d == 0]:
        for B, S in [(B, S) for B, S in [(8, 1), (7, 25), (33, 10), (1024, 3), (rb, 2), (2 * rb + 1, 5)] if B >= rb]:
            seen = torch.zeros(S, B, dtype=torch.int32)
            sizes = []
            for r in range(world):
                rs, g, k = mc.shard_layout(world, r, rb)
                assert rs * rb == world and (g, k) == (r % rs, r // rs)
                b0, b1 = mc.row_block(B, rb, k)
                sizes.append(b1 - b0)
                for j in mc.local_samples(S, rs, g):
                    seen[j, b0:b1] += 1
            assert bool((seen == 1).all()), (world, rb, B, S)
            assert max(sizes) - min(sizes) <= 1 and min(sizes) >= 1
            # ragged blocks: the first B % rb blocks are the longer ones
            blocks = [mc.row_block(B, rb, k) for k in range(rb)]
            assert [b1 - b0 for b0, b1 in blocks] == sorted((b1 - b0 for b0, b1 in blocks), reverse=True)
            assert blocks[0][0] == 0 and blocks[-1][1] == B
    with pytest.raises(Exception):
        mc.shard_layout(6, 0, 4)


def test_desc_encodes_the_first_image(built):
    from pytorch_bayesiancnn_b200 import _lib as L, functional as Fn
    args = ((16, 3, 32, 32), (64, 3, 5, 5), ((1, 1), (2, 2), (1, 1)), L.VARIANT_LRT, True, True, 0.0, 0.1, L.MATH_BF16_TC)
    assert list(Fn.make_desc(*args).reserved) == [0, 0, 0, 0]
    d = Fn.make_desc(*args, first_image=300)
    assert list(d.reserved) == [300 << 8, 0, 0, 0]
    d = Fn.make_desc(*args, fold=(8, 3 << 40), first_image=Fn.FIRST_IMAGE_MAX)
    assert d.reserved[0] == Fn.FIRST_IMAGE_MAX << 8 and d.reserved[1] == 8 and d.reserved[3] == 3 << 8
    assert (d.reserved[0] & 0xFF) == 0 and d.reserved[0] > 0            # bits 0..1 stay free for the fused phase
    with pytest.raises(L.EngineError):
        with Fn.first_image(-1):
            pass
    with pytest.raises(L.EngineError):
        with Fn.first_image(Fn.FIRST_IMAGE_MAX + 1):
            pass
    with Fn.first_image(7):
        assert Fn.current_first_image() == 7
    assert Fn.current_first_image() == 0


def test_support_queries_accept_and_refuse_the_first_image(built):
    from pytorch_bayesiancnn_b200 import _lib as L, functional as Fn
    lib = L.lib()
    conv = ((1, 1), (2, 2), (1, 1))
    for math in (L.MATH_FP32, L.MATH_BF16_TC, L.MATH_TF32_TC):
        for variant in (L.VARIANT_LRT, L.VARIANT_BBB):
            d = Fn.make_desc((16, 3, 32, 32), (64, 3, 5, 5), conv, variant, True, True, 0.0, 0.1, math, first_image=1000)
            assert lib.bbb_forward_supported(ctypes.byref(d)) == 0, lib.bbb_last_error()
            d.reserved[0] = -256                                        # a negative first image
            assert lib.bbb_forward_supported(ctypes.byref(d)) == -1
            assert b"negative" in lib.bbb_last_error()
            # (first image + batch) x OH*OW x Cout past int32 element counts: 32x32x64 outputs per image
            d.reserved[0] = Fn.first_image_word((1 << 31) // (32 * 32 * 64) - 16 + 1)
            assert lib.bbb_forward_supported(ctypes.byref(d)) == -1
            assert b"int32" in lib.bbb_last_error()
            d.reserved[0] = Fn.first_image_word((1 << 31) // (32 * 32 * 64) - 16 - 1)
            assert lib.bbb_forward_supported(ctypes.byref(d)) == 0
    # a fold counts its rows per sample, not the folded batch
    d = Fn.make_desc((4 * 128, 3, 32, 32), (64, 3, 5, 5), conv, L.VARIANT_LRT, True, True, 0.0, 0.1, L.MATH_BF16_TC,
                     fold=(128, 1 << 40), first_image=(1 << 31) // (32 * 32 * 64) - 200)
    assert lib.bbb_forward_supported(ctypes.byref(d)) == 0, lib.bbb_last_error()
    # the fused chain: first image beside the phase bits
    from pytorch_bayesiancnn_b200 import fused, models
    net = models.BBBAlexNet(10, 3, CFG_PRIORS, "lrt", "softplus")
    net.set_flag("math", "bf16")
    with Fn.first_image(500):
        steps = fused.plan(list(net.children()), (256, 3, 32, 32))
        assert steps is not None
        for st in steps:
            d = fused._step_desc(st, L.FUSED_SKIP_PREP)
            assert d.reserved[0] == (500 << 8) | L.FUSED_SKIP_PREP
            rc = lib.bbb_fused_supported(ctypes.byref(d), st.in_layout, fused._in_pitch(st), st.prev_hw, st.out_layout,
                                         fused._out_pitch(st))
            assert rc == 0, lib.bbb_last_error()
            d.reserved[0] = -1
            assert lib.bbb_fused_supported(ctypes.byref(d), st.in_layout, fused._in_pitch(st), st.prev_hw,
                                           st.out_layout, fused._out_pitch(st)) == -1
    assert list(fused._step_desc(steps[0], 0).reserved) == [0, 0, 0, 0]


def test_sharded_exchange_refuses_bad_layouts_without_gpu(built):
    from pytorch_bayesiancnn_b200 import _lib as L
    lib = L.lib()
    peers = (ctypes.c_void_p * 4)(*([1] * 4))
    common = lambda world, rb, B: lib.bbb_mc_exchange_sharded(
        None, 0, 1, B, 10, None, 0, 0, None, ctypes.c_float(1.0), ctypes.c_float(0.0), 0, world, peers, ctypes.c_void_p(1),
        ctypes.c_void_p(1), None, None, None, None, None, None, None, 0, None, None, rb, None)
    assert common(4, 3, 16) == -1 and b"multiple" in lib.bbb_last_error()
    assert common(4, 4, 3) == -1 and b"empty" in lib.bbb_last_error()
    assert common(4, 0, 16) == -1


# --------------------------------------------------------------------------- #
# the generic path over gloo: batch_shards in {1, 2, 4} on 4 processes
# --------------------------------------------------------------------------- #
def _forward_fn():
    from oracle import bbb_oracle as O
    params = O.init_params("lenet", 10, 3, CFG_PRIORS, seed=5)
    B = 7
    shapes = O.eps_shapes("lenet", 10, 3, "lrt", B)

    def fn(x, j):
        # activation noise of the whole batch keyed by the GLOBAL sample id; a row block takes its images' rows
        from pytorch_bayesiancnn_b200 import functional as Fn
        b0 = Fn.current_first_image()
        eps = [e[b0:b0 + x.shape[0]] for e in O.draw_eps_like_reference(shapes, seed=1000 + j)]
        return O.net_forward("lenet", params, x, eps, "lrt", "softplus", 0.0, 0.1, 10)
    return fn


def _worker(rank, world, port, num_ens, out_path):
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"; os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    torch.set_num_threads(1)
    from pytorch_bayesiancnn_b200 import mc
    x = torch.randn(7, 3, 32, 32, generator=torch.Generator().manual_seed(0))
    res = {}
    for rb in (1, 2, 4):
        res[rb] = mc.mc_forward(_forward_fn(), x, num_ens, want_uncertainty=True, information=True, batch_shards=rb)
    torch.save(res, out_path + f".{rank}")
    dist.destroy_process_group()


@pytest.mark.parametrize("num_ens", [1, 5])
def test_generic_path_is_independent_of_batch_shards(num_ens):
    from oracle import bbb_oracle as O
    from pytorch_bayesiancnn_b200 import mc
    torch.set_num_threads(1)
    x = torch.randn(7, 3, 32, 32, generator=torch.Generator().manual_seed(0))
    fn = _forward_fn()
    logits = [fn(x, j) for j in range(num_ens)]
    ref = O.mc_combine([l for l, _ in logits])
    single = mc.mc_forward(fn, x, num_ens, want_uncertainty=True, information=True)
    assert torch.allclose(single[0], ref, atol=1e-5)
    world = 4
    s = socket.socket(); s.bind(("127.0.0.1", 0)); port = s.getsockname()[1]; s.close()
    out_path = os.path.join(tempfile.mkdtemp(), "rank")
    ctx = mp.get_context("spawn")
    procs = [ctx.Process(target=_worker, args=(r, world, port, num_ens, out_path)) for r in range(world)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(timeout=300)
        assert p.exitcode == 0
    outs = [torch.load(out_path + f".{r}") for r in range(world)]
    for rb in (1, 2, 4):
        lo, kl, unc = outs[0][rb]
        for o in outs[1:]:                                  # every rank returns the same full outputs
            assert torch.equal(o[rb][0], lo) and all(torch.equal(a, b) for a, b in zip(o[rb][2], unc))
        assert lo.shape == (7, 10) and torch.allclose(lo, ref, atol=1e-5), rb
        assert abs(float(kl) - float(logits[0][1])) <= 1e-6 * abs(float(kl)), rb      # each group's KL counted once
        for a, b in zip(unc, single[2]):
            assert torch.allclose(a, b, atol=1e-6), rb
        if rb > 1:                                          # the same numbers whatever the split
            for a, b in zip(unc, outs[0][1][2]):
                assert torch.allclose(a, b, atol=1e-6)
