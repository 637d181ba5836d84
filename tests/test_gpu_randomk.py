"""The fused engine's 'randomk' mode (shared-seed index, values only on the wire) on the GPU, against the oracle.

W = 1 through ``test_gpu_engine._run_vs_oracle``; W = 2, 4, 8 through the one-GPU W-rank harness of
``test_engine_multirank`` (sharded, unsharded and the NCCL transport); the fallback phase under a bound that is too
tight; the receiver's agreement check (status 7); and the benchmark's training step against plain torch +
``engine_oracle``."""
import numpy as np
import pytest
import torch

import bench
import test_engine_multirank as multirank
import test_gpu_engine as single
from deepreduce_b200.parallel import BucketEngine, BucketPlan, engine_oracle
from deepreduce_b200.parallel.engine import PH_ACCUM, PH_END, PH_INSERT, PH_SIGNAL, PH_SIGNAL2
from deepreduce_b200.parallel.plan import DYN_WORDS, KEY_SPAN, MODE_SHARED, SLOT_HEADER_WORDS
from test_gpu_engine import SIZES, _fill
from test_train_step_reference import run_case

pytestmark = pytest.mark.gpu

BIG = SIZES + [2359296]


def _compare_shared_slot(plan, slot_gpu, slot_ref, tag):
    """Slot comparison for MODE_SHARED tensors: header and dyn words exact; fp32 values word for word; QSGD norms to
    fp32 rounding and levels up to the rounding-boundary flips ``test_gpu_engine._compare_slot`` allows."""
    a = slot_gpu.cpu().numpy().view(np.uint32)
    b = slot_ref
    bad = []
    if not np.array_equal(a[:5], b[:5]):
        bad.append(f"header {a[:5]} vs {b[:5]}")
    for ti, t in enumerate(plan.tensors):
        assert t.mode == MODE_SHARED
        d0 = SLOT_HEADER_WORDS + DYN_WORDS * ti
        if not np.array_equal(a[d0:d0 + 4], b[d0:d0 + 4]):
            bad.append(f"{t.name} dyn gpu={a[d0:d0 + 4].tolist()} ref={b[d0:d0 + 4].tolist()}")
        n = int(b[d0])
        if t.vmode == 2:
            nb = (n + 511) // 512
            na, nr = a[t.off_coef:t.off_coef + nb].view(np.float32), b[t.off_coef:t.off_coef + nb].view(np.float32)
            if not np.allclose(na, nr, rtol=1e-5):
                bad.append(f"{t.name} qsgd norms differ {float(np.abs(na - nr).max())}")
            dt, per = (np.int16, 2) if t.rank_u32 else (np.int8, 4)
            la = a[t.off_rankmap:t.off_rankmap + (n + per - 1) // per].view(dt)[:n]
            lr = b[t.off_rankmap:t.off_rankmap + (n + per - 1) // per].view(dt)[:n]
            if int((la != lr).sum()) > max(2, n // 2000):
                bad.append(f"{t.name} qsgd levels differ in {int((la != lr).sum())}/{n}")
        elif not np.array_equal(a[t.off_vals:t.off_vals + n], b[t.off_vals:t.off_vals + n]):
            bad.append(f"{t.name} vals differ in {int((a[t.off_vals:t.off_vals + n] != b[t.off_vals:t.off_vals + n]).sum())}/{n}")
    # nothing else is shipped: the whole payload matches word for word when the values are fp32
    if not any(t.vmode for t in plan.tensors) and not np.array_equal(a[:plan.payload_words], b[:plan.payload_words]):
        bad.append("payload words differ outside the per-tensor regions")
    return bad


@pytest.mark.parametrize("tma", [True, False])
@pytest.mark.parametrize("value", [None, "qsgd"])
def test_randomk_single_rank_vs_oracle(monkeypatch, tma, value):
    """W = 1 with residual, three epochs (the second through the unfused phase chain), every size class of
    ``test_gpu_engine``: slots, dense output and residual bit-exact for fp32, QSGD within that helper's tolerances."""
    monkeypatch.setattr(single, "_compare_slot", _compare_shared_slot)
    for kind in ("randn", "sparse"):
        single._run_vs_oracle(kind, None, "leftmost", True, tma, value, sparsifier="randomk")


@pytest.mark.parametrize("value,bps", [(None, 2), (None, 1), ("qsgd", 2)])
def test_randomk_single_rank_without_residual(value, bps):
    plan = BucketPlan(BIG, compress_ratio=0.01, index=None, value=value, sparsifier="randomk")
    eng = BucketEngine(plan, device="cuda:0", world=1, rank=0, beta=0.0, spin_limit=2_000_000, blocks_per_sm=bps)
    gen = torch.Generator().manual_seed(3)
    zero = torch.zeros(plan.total_elems)
    for step in range(4):
        g = _fill(plan, gen)
        eng.grad.copy_(g.cuda())
        eng.step()
        torch.cuda.synchronize()
        eng.check_status()
        out_ref, new_res, slots = engine_oracle(plan, [g], [zero], beta=0.0, epoch=eng.epoch)
        bad = _compare_shared_slot(plan, eng.slot(), slots[0], f"randomk_nores_{value}_s{step}")
        assert not bad, bad[:4]
        if value is None:
            assert torch.equal(eng.grad.cpu(), out_ref) and torch.equal(eng.resid.cpu(), new_res[0])
        else:
            sc = float(out_ref.abs().max())
            assert torch.allclose(eng.grad.cpu(), out_ref, atol=2e-3 * sc, rtol=1e-2)
            assert torch.allclose(eng.resid.cpu(), new_res[0], atol=2e-3 * sc, rtol=1e-2)
    eng.close()


def test_randomk_fallback_under_a_tight_bound():
    """A static bound above the threshold hides it: the accumulate phase flags the tensors, phase 1 rebuilds the
    candidate lists from the index hashes (not from the residual's bits), and the step still matches the oracle."""
    plan = BucketPlan(BIG, compress_ratio=0.01, index=None, sparsifier="randomk")
    for t in plan.tensors:
        t.shared_lb = (KEY_SPAN - 4096) & ~511                 # ~numel / 2^19 candidates: fewer than K everywhere
    eng = BucketEngine(plan, device="cuda:0", world=1, rank=0, beta=0.0, spin_limit=2_000_000)
    gen = torch.Generator().manual_seed(4)
    for epoch in (1, 2, 3):
        g = _fill(plan, gen)
        # first the select phases alone, to read how many tensors needed the fallback
        eng.grad.copy_(g.cuda())
        eng.barrier.zero_()
        eng.run_phases(PH_ACCUM, PH_INSERT, epoch)
        torch.cuda.synchronize()
        eng.check_status()
        n_unsafe = int(eng.barrier[8].item())
        assert n_unsafe >= len(plan.tensors) - 2, n_unsafe   # the two tiniest tensors may still hold K candidates
        # then the whole step on the same epoch, from clean select scratch
        eng.hist.zero_(); eng.hist_total.zero_(); eng.tile_count.zero_(); eng.barrier.zero_()
        eng.grad.copy_(g.cuda())
        eng.step(epoch)
        torch.cuda.synchronize()
        eng.check_status()
        out_ref, new_res, slots = engine_oracle(plan, [g], [torch.zeros_like(g)], beta=0.0, epoch=epoch)
        bad = _compare_shared_slot(plan, eng.slot(), slots[0], f"randomk_fallback_e{epoch}")
        assert not bad, bad[:4]
        assert torch.equal(eng.grad.cpu(), out_ref) and torch.equal(eng.resid.cpu(), new_res[0])
    eng.close()


# (configuration, W, plan keyword arguments, DR_DETERMINISTIC, average)
MULTI = [
    pytest.param("shard", 2, {}, False, True, id="shard-W2-fast"),
    pytest.param("shard", 4, {}, False, True, id="shard-W4-fast"),
    pytest.param("shard", 8, {}, True, False, id="shard-W8-det-sum"),
    pytest.param("shard", 4, dict(value="qsgd"), False, True, id="shard-qsgd8-W4-fast"),
    pytest.param("shard", 8, dict(value="qsgd", quantum_num=1000), True, True, id="shard-qsgd16-W8-det"),
    pytest.param("noshard", 2, {}, False, True, id="noshard-W2-fast"),
    pytest.param("noshard", 4, dict(value="qsgd"), False, False, id="noshard-qsgd8-W4-fast-sum"),
    pytest.param("noshard", 8, {}, False, True, id="noshard-W8-fast"),
    pytest.param("nccl", 2, dict(value="qsgd"), False, True, id="nccl-qsgd8-W2-fast"),
    pytest.param("nccl", 4, {}, True, True, id="nccl-W4-det"),
    pytest.param("nccl", 8, {}, False, False, id="nccl-W8-fast-sum"),
]


@pytest.mark.timeout(900)
@pytest.mark.parametrize("config,W,kw,deterministic,average", MULTI)
def test_randomk_multirank_vs_oracle(monkeypatch, config, W, kw, deterministic, average):
    """W ranks on one GPU: slots and residuals against ``engine_oracle``, delivery of every slot, the aggregate
    against the rank-ordered sum of the decoded slots (bit for bit for fp32, as plain pairs are), identical bits on
    every rank, and the stage-2 lists (``test_engine_multirank_vs_oracle`` with the shared-index slot comparison)."""
    monkeypatch.setattr(multirank, "_compare_slot", _compare_shared_slot)
    sizes = multirank.BIG if config == "shard" and W == 2 else SIZES
    multirank.test_engine_multirank_vs_oracle(monkeypatch, config, W, sizes, dict(index=None, sparsifier="randomk", **kw),
                                              deterministic, average, None, set())


@pytest.mark.parametrize("config", ["shard", "noshard"])
def test_randomk_disagreeing_sender_is_status_7(monkeypatch, config):
    """A sender whose header words differ from the receiver's own drew another set: the receiver reports status 7
    and leaves that sender out.  The header is edited in the receiver's arena between the push and the decode."""
    monkeypatch.setenv("DR_DETERMINISTIC", "0")
    W = 2
    plan = BucketPlan(BIG, compress_ratio=0.01, index=None, sparsifier="randomk")
    engs = multirank._engines(plan, W, config, True)
    gen = torch.Generator().manual_seed(9)
    grads = [_fill(plan, gen) for _ in range(W)]
    epoch = 1
    for e, g in zip(engs, grads):
        e.grad.copy_(g.cuda())
    multirank._wave(engs, PH_ACCUM, PH_SIGNAL, epoch)
    ti = len(plan.tensors) - 1                                  # the big tensor: tiles in both ranks' slices
    t = plan.tensors[ti]
    w = SLOT_HEADER_WORDS + DYN_WORDS * ti + 2
    recv = engs[1]
    recv.slot(0, epoch)[w] += 512                               # sender 0's threshold, as rank 1 received it
    # sharded: stop in front of the stage-2 flag wait (the engines of a wave run one after the other, so rank 0 would
    # wait for stage-2 flags that rank 1 releases only in its own launch); unsharded: there is no second wait
    end = PH_SIGNAL2 if config == "shard" else PH_END
    for e in engs:
        e.run_phases(PH_SIGNAL, end, epoch)
    torch.cuda.synchronize()
    st0, st1 = engs[0].status.cpu().tolist(), recv.status.cpu().tolist()
    assert st0[0] == 0, st0
    assert st1[0] == 7 and st1[1] == 0, st1
    # the receiver's part of the big tensor holds its own contribution only
    out_ref, _, slots = engine_oracle(plan, [grads[1]], [torch.zeros_like(grads[1])], epoch=epoch)
    lo, hi = (multirank._spans(plan.n_tiles, W)[1] if config == "shard" else (0, plan.n_tiles))
    first = max(lo, t.tile_begin)
    last = min(hi, t.tile_begin + t.n_tiles)
    seg = slice(t.elem_off + (first - t.tile_begin) * 4096, min(t.elem_off + t.numel, t.elem_off + (last - t.tile_begin) * 4096))
    assert torch.equal(recv.grad.cpu()[seg], out_ref[seg] / W)
    for e in engs:
        e.close()


RANDOMK = {'compressor': 'randomk', 'memory': 'residual', 'compress_ratio': 0.01}


@pytest.mark.timeout(900)
@pytest.mark.parametrize("communicator", ["allgather", "allreduce"])
def test_resnet50_randomk_train_step(monkeypatch, communicator):
    """ResNet-50, batch 16, three steps of the benchmark's ``Trainer`` with 'randomk' against plain torch +
    ``engine_oracle``, bit for bit: loss, bucket, residual, parameters, momentum and BatchNorm buffers."""
    monkeypatch.setitem(bench.CONFIGS, "randomk", {**RANDOMK, 'communicator': communicator})

    def check(tr):
        assert tr.ddp.fused and tr.ddp.grc is None
        assert all(t.mode == MODE_SHARED for e in tr.ddp.engines for t in e.plan.tensors)
    run_case(monkeypatch, "image", "randomk", 16, check=check)
