"""The fused gradient exchange (csrc/comm_kernels.cu) at world sizes 1 to 16 on one GPU: W stand-in ranks (tests/dev/comm_dev.cu,
the product's machine code) step one after another on one stream, and after every step each is held to the references of
tests/dev/comm_ranks.py: the reduced gradient bit for bit against the float32 restatement of the rank-order sum and within its
bound of the float64 mean, the two norms and clip coefficients, float64 Adam on the device's own gradient, identical replicas,
the flag and state words, the gradients and buffer tails nothing may write, graph replay, the adaptive rate over the ranks' KLs
and the bounded wait for a peer that never arrives."""
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "dev"))
import comm_ranks as CR  # noqa: E402

pytestmark = pytest.mark.gpu
NETS = CR.network_sizes()
SIZES = ["1", "3", "4", "5", "1703"] + list(NETS) + ["grid_cap"]
REGIMES = [(True, True), (False, False), (True, False), (False, True)]     # (actor clipped, critic clipped)
WORST = {}


def _size(name):
    if name == "grid_cap":
        return CR.grid_cap_size(torch.cuda.get_device_properties(0).multi_processor_count), None
    return NETS[name] if name in NETS else (int(name), None)


def _note(key, x):
    WORST[key] = max(WORST.get(key, 0.0), float(x))


def _round(R, n_actor, hp, kls=None):
    """Every rank's step in rank order; after rank r's: every rank's flag word for r is epoch + 1 (W > 1: at W = 1 there is
    no flag traffic) and r's state is {epoch + 2, 0, 0, step + 1}."""
    e, s = (int(x) for x in R.state[0][[CR.ST_EPOCH, CR.ST_STEP]].cpu())
    kl = None if kls is None else [torch.tensor([k], dtype=torch.float32, device="cuda") for k in kls]
    if kls is not None:
        R.set_kl_words(kls)
    for r in range(R.world):
        R.step(r, n_actor, hp, None if kl is None else kl[r])
        want = [e + 1] * R.world if R.world > 1 else [0]
        assert [int(R.flags[q][r]) for q in range(R.world)] == want, (r, e)
        assert R.state[r].cpu().tolist() == [e + 2, 0, 0, s + 1], (r, R.state[r].cpu().tolist(), e, s)


def _check_step(R, gs, n_actor, before, clipped):
    """The checks after one round of a fixed-rate step; `before`: rank 0's host buffers before it."""
    n, W, hp = R.n, R.world, CR.HP
    h = [R.host(r) for r in range(W)]
    for r in range(1, W):            # replicas: every buffer, sentinel tails included, and every rank's copy of the Adam step
        for k in ("p", "m", "v", "reduced", "coef"):
            assert np.array_equal(CR.bits(h[r][k]), CR.bits(h[0][k])), (k, r)
    for r in range(W):               # no rank wrote into any peer's gradient or past n_total
        assert np.array_equal(CR.bits(R.grad[r][:n].cpu().numpy()), CR.bits(gs[r])), r
    for k in ("p", "m", "v", "reduced"):
        assert np.all(CR.bits(h[0][k][n:]) == CR.SENTINEL), k
    red, coef = h[0]["reduced"][:n], h[0]["coef"]
    # 1. the specified reduction bit for bit, and within its bound of the float64 mean
    want = CR.reduce_f32(gs)
    bad = np.flatnonzero(CR.bits(red) != CR.bits(want))
    assert bad.size == 0, (bad[:5], red[bad[:5]], want[bad[:5]])
    err, bound = np.abs(red.astype(np.float64) - gs.astype(np.float64).mean(0)), CR.reduce_bound(gs)
    assert np.all(err <= bound)
    _note("reduced / bound", np.max(err / np.maximum(bound, 1e-300)))
    # 2. the norms over each network's elements of the average, and the clip coefficients from them
    for t_dev, t64, c_dev in zip(coef[2:4], CR.norms64(red, n_actor), coef[0:2]):
        ref = np.float32(t64)
        assert abs(float(t_dev) - float(ref)) <= float(np.spacing(ref)), (t_dev, t64)
        _note("norm / ulp", abs(float(t_dev) - t64) / float(np.spacing(ref)))
        assert CR.bits(c_dev) == CR.bits(CR.clip_coef(t_dev, hp["max_norm"])), (c_dev, t_dev)
    segs = [(0, n_actor), (n_actor, n)]
    assert [bool(c < 1) for c, (lo, hi) in zip(coef[:2], segs) if hi > lo] == [c for c, (lo, hi) in zip(clipped, segs) if hi > lo]
    # 3. float64 Adam on the device's own reduced gradient and clip coefficients
    t = int(before["state"][CR.ST_STEP]) + 1
    p, m, v = CR.adam64(before["p"][:n], before["m"][:n], before["v"][:n], red, coef[0], coef[1], n_actor, t, hp)
    dp = np.abs(h[0]["p"][:n] - p) / (CR.ulp32(p) + CR.PARAM_LR * float(np.float32(hp["lr"])))
    assert dp.max() <= 1.0, dp.max()
    _note("param / allowance", dp.max())
    for got, ref in ((h[0]["m"][:n], m), (h[0]["v"][:n], v)):
        for lo, hi in segs:
            if hi > lo and np.linalg.norm(ref[lo:hi]) > 0:
                rel = np.linalg.norm(got[lo:hi] - ref[lo:hi]) / np.linalg.norm(ref[lo:hi])
                assert rel <= CR.MOMENT_BOUND, rel
                _note("moments / bound", rel / CR.MOMENT_BOUND)


@pytest.mark.parametrize("size", SIZES)
@pytest.mark.parametrize("W", CR.WORLDS)
def test_each_step_matches_the_references(W, size):
    n, boundary = _size(size)
    splits = CR.actor_splits(n, boundary)
    if boundary is not None or size == "grid_cap":
        splits = [boundary if boundary is not None else n // 2, 0, n]
    rng = np.random.default_rng(1000 * W + n)
    R = CR.Ranks(n, W, rng.standard_normal(n).astype(np.float32))
    try:
        for k in range(max(4, len(splits))):
            n_actor, clipped = splits[k % len(splits)], REGIMES[k % len(REGIMES)]
            gs = CR.scaled_grads(rng, W, n, n_actor, clipped, CR.HP["max_norm"])
            R.set_grads(gs)
            before = R.host(0)
            _round(R, n_actor, CR.HP)
            _check_step(R, gs, n_actor, before, clipped)
    finally:
        R.close()


@pytest.mark.parametrize("adaptive", [False, True], ids=["fixed", "adaptive"])
@pytest.mark.parametrize("W", [2, 5, 16])
def test_graph_replay_is_the_eager_sequence(W, adaptive):
    """The W ranks' steps captured once in one graph, the flag presets as memset nodes; the epoch and the Adam step come from
    device memory on every replay."""
    n, n_actor = 1703, 1001
    rng = np.random.default_rng(W)
    p0 = rng.standard_normal(n).astype(np.float32)
    E, G = CR.Ranks(n, W, p0), CR.Ranks(n, W, p0)
    kl = [torch.zeros(1, device="cuda") for _ in range(W)]
    for R in (E, G):
        for r in range(W):
            R.lr[r].fill_(3e-4)
    try:
        torch.cuda.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            for r in range(W):
                G.step(r, n_actor, CR.HP, kl[r] if adaptive else None)
        assert G.state[0].cpu().tolist() == [1, 0, 0, 0]           # capture does not run the step
        cases = CR.kl_cases(W)
        for k in range(5):
            gs = CR.scaled_grads(rng, W, n, n_actor, REGIMES[k % 4], CR.HP["max_norm"])
            kls = cases[k % len(cases)][1]
            for r in range(W):
                kl[r].fill_(float(kls[r]))
            for R in (E, G):
                R.set_grads(gs)
                if adaptive:
                    R.set_kl_words(kls)
            for r in range(W):
                E.step(r, n_actor, CR.HP, kl[r] if adaptive else None)
            graph.replay()
            for r in range(W):
                he, hg = E.host(r), G.host(r)
                for key in he:
                    assert np.array_equal(he[key].view(np.uint8), hg[key].view(np.uint8)), (k, r, key)
                assert E.lr[r].cpu().numpy().tobytes() == G.lr[r].cpu().numpy().tobytes(), (k, r)
        assert G.state[0].cpu().tolist() == [11, 0, 0, 5]
    finally:
        E.close()
        G.close()


@pytest.mark.parametrize("W", CR.WORLDS)
def test_adaptive_rate_is_the_host_rule_on_the_rank_order_mean(W):
    """Distinct KLs per rank (thresholds, a NaN on one rank, an order-dependent float64 sum): after every step every rank's rate
    is adapt_lr(rate, rank_mean_kl(kls), D) bit for bit, and the parameters and moments are those of the fixed-rate exchange
    run at that rate."""
    from learninghumanoidwalking_b200.rl.schedule import adapt_lr, rank_mean_kl
    n, n_actor = 1703, 702
    rng = np.random.default_rng(50 + W)
    p0 = rng.standard_normal(n).astype(np.float32)
    A, F = CR.Ranks(n, W, p0), CR.Ranks(n, W, p0)
    try:
        lr = 3e-4
        for r in range(W):
            A.lr[r].fill_(lr)
        for k, (name, kls, move) in enumerate(CR.kl_cases(W)):
            gs =CR.scaled_grads(rng, W, n, n_actor, REGIMES[k % 4], CR.HP["max_norm"])
            A.set_grads(gs)
            F.set_grads(gs)
            _round(A, n_actor, CR.HP, kls)
            want = adapt_lr(lr, rank_mean_kl(kls), CR.D)
            got = [float(A.lr[r].item()) for r in range(W)]
            assert all(np.float64(g).tobytes() == np.float64(want).tobytes() for g in got), (name, kls, got, want)
            assert {"up": want > lr, "down": want < lr, "same": want == lr}[move], (name, lr, want)
            _round(F, n_actor, dict(CR.HP, lr=float(np.float32(want))))
            for r in range(W):
                ha, hf = A.host(r), F.host(r)
                for key in ("p", "m", "v", "reduced", "coef"):
                    assert np.array_equal(CR.bits(ha[key]), CR.bits(hf[key])), (name, r, key)
            lr = want
    finally:
        A.close()
        F.close()


@pytest.mark.parametrize("W,late", [(2, 0), (4, 2)])
def test_a_peer_that_never_arrives_leaves_an_error_word(W, late):
    """Rank `late` steps with its last peer's flag word behind the epoch and a spin limit of 2^10 polls: both waits give up
    after about a millisecond, the step completes, and the status call reports error word 3 (ready and done time-outs)."""
    n = 1703
    rng = np.random.default_rng(7)
    R = CR.Ranks(n, W, rng.standard_normal(n).astype(np.float32))
    try:
        R.set_grads(CR.scaled_grads(rng, W, n, 700, (False, False), CR.HP["max_norm"]))
        for r in range(late):
            R.step(r, 700, CR.HP)
        R.set_spin_limit(late, 2 ** 10)
        assert int(R.flags[late][W - 1]) == 0 < int(R.state[late][CR.ST_EPOCH])
        R.step(late, 700, CR.HP, preset=False)
        rc, err, steps, _, msg = R.status(late)
        assert (rc, err, steps) == (-20, 3, 1), (rc, err, steps, msg)
        assert "peer exchange timed out (error word 3)" in msg
        assert R.state[late].cpu().tolist() == [3, 3, 0, 1]
        for r in range(late):
            assert R.status(r)[:2] == (0, 0)
    finally:
        R.close()


def test_report_largest_ratios():
    """Run last in this module: prints the largest error-to-bound ratios the cases above met."""
    print("\n[exchange ranks] largest ratios: " + ", ".join(f"{k} {v:.3g}" for k, v in sorted(WORST.items())))
