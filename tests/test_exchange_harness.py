"""The stand-in ranks of the fused gradient exchange without a GPU: the device harness (tests/dev/comm_dev.cu) cross-compiles for
sm_90a with the product's machine code for every exchange kernel and exports only its own entry points, and the references
tests/test_gpu_exchange_ranks.py holds the kernels to (tests/dev/comm_ranks.py) check themselves."""
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "dev"))
import comm_ranks as CR  # noqa: E402


def test_harness_runs_the_product_sass_function_by_function():
    dev, prod = CR.sass_functions(CR.build_harness()), CR.sass_functions(CR.build_product())
    assert sorted(dev) == sorted(prod) and len(dev) == len(CR.KERNELS), (sorted(dev), sorted(prod))
    for k in CR.KERNELS:
        (name,) = [f for f in dev if k in f]
        assert dev[name] == prod[name], name
        assert len(dev[name]) > 50


def test_harness_exports_only_its_entry_points():
    """Its copies of lhw_comm_create and the rest bind inside it and cannot shadow liblhw_b200.so's in the same process."""
    out = subprocess.run(["nm", "-D", "--defined-only", CR.build_harness()], capture_output=True, text=True, check=True).stdout
    names = {line.split()[-1] for line in out.splitlines() if line.strip()}
    assert names == {"cx_create", "cx_destroy", "cx_pointers", "cx_set_spin_limit", "cx_preset_later_peers", "cx_step",
                     "cx_step_adaptive", "cx_status", "cx_last_error"}, names


@pytest.mark.parametrize("W", CR.WORLDS)
def test_float32_restatement_is_within_its_bound_of_the_float64_mean(W):
    rng = np.random.default_rng(W)
    n = 20000
    gs = (rng.standard_normal((W, n)) * np.exp(rng.uniform(-20, 20, (W, n)))).astype(np.float32)
    gs[:, :100] = -gs[0, :100]                   # heavy cancellation where W is even
    red = CR.reduce_f32(gs)
    err = np.abs(red.astype(np.float64) - gs.astype(np.float64).mean(0))
    bound = CR.reduce_bound(gs)
    assert red.dtype == np.float32 and np.all(err <= bound), float(np.max(err / np.maximum(bound, 1e-300)))
    if W > 2:
        assert np.any(err > 0)
    # a sum started at +0.0f turns -0.0 on every rank into +0.0; one started at g_0 would keep -0.0, which == hides
    z = np.full((W, 1), -0.0, np.float32)
    from_g0 = z[0]
    for g in z[1:]:
        from_g0 = from_g0 + g
    assert CR.bits(CR.reduce_f32(z))[0] == 0 and CR.bits(from_g0 / np.float32(W))[0] == 0x80000000


@pytest.mark.parametrize("W", CR.WORLDS)
def test_kl_sets_move_the_rate_as_named(W):
    from learninghumanoidwalking_b200.rl.schedule import adapt_lr, rank_mean_kl
    cases = {name: (kls, move) for name, kls, move in CR.kl_cases(W)}
    assert len({float(k) for k in cases["above_2D"][0]}) == W
    assert rank_mean_kl(cases["on_2D"][0]) == 2 * CR.D and rank_mean_kl(cases["on_D/2"][0]) == CR.D / 2
    assert math.isnan(rank_mean_kl(cases["nan_on_one_rank"][0]))
    if W >= 4:
        kls = cases["order"][0]
        assert rank_mean_kl(kls) > 0 and rank_mean_kl(kls[::-1]) == 0.0
        assert adapt_lr(3e-4, rank_mean_kl(kls), CR.D) > 3e-4 and adapt_lr(3e-4, rank_mean_kl(kls[::-1]), CR.D) == 3e-4


def test_clip_coefficient_is_clip_grad_norm_in_float32():
    for t in (0.0, 1e-7, 0.3, 0.69999, 0.7, 0.7000001, 2.1, 1e6):
        p = torch.nn.Parameter(torch.zeros(1))
        p.grad = torch.tensor([t], dtype=torch.float32)
        torch.nn.utils.clip_grad_norm_([p], 0.7)
        want = np.float32(p.grad.item() / t) if t else np.float32(1)
        got = CR.clip_coef(np.float32(t), 0.7)
        assert got == min(np.float32(1), np.float32(0.7) / (np.float32(t) + np.float32(1e-6)))
        if t:
            assert abs(float(got) - float(want)) <= 2 * float(np.spacing(got)), (t, got, want)


def test_float64_adam_is_torch_adam_after_clip():
    rng = np.random.default_rng(3)
    n, n_actor, hp = 50, 20, CR.HP
    p = rng.standard_normal(n).astype(np.float32)
    m = v = np.zeros(n, np.float32)
    ta, tc = (torch.tensor(x, dtype=torch.float64, requires_grad=True) for x in (p[:n_actor], p[n_actor:]))
    f = lambda k: float(np.float32(hp[k]))
    opts = [torch.optim.Adam([x], lr=f("lr"), betas=(f("b1"), f("b2")), eps=f("eps")) for x in (ta, tc)]
    for t in range(1, 4):
        red = (rng.standard_normal(n) * (1.0 if t == 2 else 0.01)).astype(np.float32)
        ca, cc = (CR.clip_coef(np.float32(x), hp["max_norm"]) for x in CR.norms64(red, n_actor))
        p, m, v = CR.adam64(p, m, v, red, ca, cc, n_actor, t, hp)
        for x, g, c, o in ((ta, red[:n_actor], ca, opts[0]), (tc, red[n_actor:], cc, opts[1])):
            x.grad = torch.tensor(g, dtype=torch.float64) * float(c)
            o.step()
        assert np.allclose(p, np.concatenate([ta.detach().numpy(), tc.detach().numpy()]), rtol=1e-13, atol=1e-15)


def test_sizes_come_from_the_networks():
    sizes = CR.network_sizes()
    assert sizes["jvrc_walk"] == (154381, 78604)          # SURVEY Appendix B: the reference's actor + critic
    assert sizes["jvrc_walk_learn_std"] == (154393, 78616)
    assert any(n % 4 for n, _ in sizes.values())
    assert CR.grid_cap_size(132) % 4 == 3
    for n in (1, 3, 4, 5, 1703):
        s = CR.actor_splits(n)
        assert s[0] == 0 and n in s and all(0 <= a <= n for a in s)
    assert 1701 in CR.actor_splits(1703) and {0, 1, 3, 4} <= set(CR.actor_splits(4))
