"""get_state / set_state of chosen envs (pgb200_get_states / pgb200_set_states) on the GPU, device build only.

A restored env must continue exactly as the env its blob was taken from, and a restore must touch nothing but the
listed envs. Each case therefore runs handles in lockstep on the same actions: a handle that was restored against a
control handle loaded with the same blobs, and its untouched envs against a twin that never restored. Covered: a
whole-handle copy at 65 536 envs, a random half restored at 4 096 envs and in the 16-game list at 32 768, every opt-in
of the step on at once, a graph-captured handle and a host-buffer handle."""
import numpy as np
import pytest

from oracle.record import STANDIN_PACK
from oracle.ref_env import mt19937_actions

pytestmark = pytest.mark.gpu
ALL16 = "bigfish,bossfight,caveflyer,chaser,climber,coinrun,dodgeball,fruitbot,heist,jumper,leaper,maze,miner,ninja,plunder,starpilot"
KW = dict(num_levels=0, start_level=0)


def _env(n, name, **kw):
    from procgen_b200 import ProcgenGym3Env

    return ProcgenGym3Env(n, name, resource_root=STANDIN_PACK, **kw)


def _outputs(env):
    """{name: host array} of rew, rgb, first and the infos"""
    rew, ob, first = env.observe()
    out = {"rew": rew, "rgb": ob["rgb"], "first": first}
    if env._host_buffers:
        out.update(env._info)
        return {k: np.array(v) for k, v in out.items()}
    out.update(env.get_info_tensors())
    return {k: v.cpu().numpy() for k, v in out.items()}


def _assert_same(a, b, envs, when):
    for k in a:
        x, y = a[k][envs], b[k][envs]
        if not np.array_equal(x, y):
            bad = np.nonzero((x != y).reshape(len(envs), -1).any(1))[0]
            raise AssertionError(f"{when}: {k} differs at envs {np.asarray(envs)[bad[:8]]}")


def _act(envs, a):
    import torch

    t = torch.as_tensor(a, device="cuda")
    for env in envs:
        env.act(t)


def test_whole_handle_copy_coinrun_65536(product_lib):
    """200 steps, then every blob into a handle built with another rand_seed: the two run in lockstep for 64 steps"""
    n = 65536
    a = _env(n, "coinrun", distribution_mode="easy", rand_seed=0, **KW)
    acts = mt19937_actions(0, n, 264)
    for t in range(200):
        _act([a], acts[t])
    blobs = a.get_state()
    assert len(blobs) == n
    b = _env(n, "coinrun", distribution_mode="easy", rand_seed=1, **KW)
    b.set_state(blobs)
    _assert_same(_outputs(a), _outputs(b), np.arange(n), "after set_state")
    for t in range(200, 264):
        _act([a, b], acts[t])
        _assert_same(_outputs(a), _outputs(b), np.arange(n), f"step {t}")
        if t % 16 == 0:
            assert a.get_state() == b.get_state(), f"step {t}: blobs differ"
    assert a.errors() == 0 and b.errors() == 0
    a.close()
    b.close()


@pytest.mark.parametrize("name,mode,n", [("coinrun", "hard", 4096), (ALL16, "hard", 32768)])
def test_subset_restore(product_lib, name, mode, n):
    """Handle A saves every blob at t0, steps 50 times and restores a random half S from them. S then follows a control
    handle loaded with the t0 blobs; the other half follows a twin of A that never restored."""
    rng = np.random.RandomState(7)
    acts = mt19937_actions(3, n, 100)
    a = _env(n, name, distribution_mode=mode, rand_seed=0, **KW)
    twin = _env(n, name, distribution_mode=mode, rand_seed=0, **KW)
    for t in range(10):
        _act([a, twin], acts[t])
    t0 = a.get_state()
    control = _env(n, name, distribution_mode=mode, rand_seed=2, **KW)
    control.set_state(t0)
    for t in range(10, 60):
        _act([a, twin], acts[t])
    s = np.sort(rng.permutation(n)[: n // 2])
    rest = np.setdiff1d(np.arange(n), s)
    order = rng.permutation(s)  # an unsorted list
    a.set_state([t0[e] for e in order], envs=order)
    assert a.get_state(order) == [t0[e] for e in order]
    for t in range(60, 100):
        _act([a, twin, control], acts[t])
        out = _outputs(a)
        _assert_same(out, _outputs(control), s, f"step {t}, restored envs")
        _assert_same(out, _outputs(twin), rest, f"step {t}, other envs")
    blobs = a.get_state()
    assert [blobs[e] for e in s] == control.get_state(s)
    assert [blobs[e] for e in rest] == twin.get_state(rest)
    for env in (a, twin, control):
        assert env.errors() == 0
        env.close()


def test_every_opt_in(product_lib):
    """Final outputs, the pause mask, the rollout, a 4-frame consumer output and level lookahead all on: set_state
    leaves the rollout, the final outputs and the mask alone, rewrites the restored envs' current consumer frame, and
    the handle then runs in lockstep with a control without lookahead (which changes no output) that restored the same
    blobs, through resets forced with action -1: the restored envs' lookahead slots miss once, then serve."""
    import torch

    n, name = 2048, "coinrun"
    rng = np.random.RandomState(1)
    kw = dict(distribution_mode="hard", rand_seed=0, **KW)
    donor = _env(n, name, distribution_mode="hard", rand_seed=9, **KW)
    for t in range(30):
        _act([donor], mt19937_actions(5, n, 30)[t])
    blobs = donor.get_state()
    envs = [_env(n, name, **kw) for _ in range(2)]
    for i, env in enumerate(envs):
        env.final_outputs()
        env.rollout(4)
        env.enable_consumer_output(torch.float16, frames=4)
        mask = env.pause_mask()
        mask[::7] = 1
        if i == 0:
            env.enable_level_lookahead()
    a, control = envs
    acts = mt19937_actions(2, n, 120)
    for t in range(20):
        _act(envs, acts[t])
    s = rng.permutation(n)[: n // 3]
    torch.cuda.synchronize()
    before = {k: v.clone() for k, v in a.rollout(4).items()}
    final = {k: v.clone() for k, v in a.final_outputs().items()}
    stack = a.consumer_observation().clone()
    for env in envs:
        env.set_state([blobs[e] for e in s], envs=s)
    torch.cuda.synchronize()
    for k, v in a.rollout(4).items():
        assert torch.equal(v, before[k]), f"set_state changed the rollout's {k}"
    for k, v in a.final_outputs().items():
        assert torch.equal(v, final[k]), f"set_state changed the final outputs' {k}"
    assert int(a.pause_mask().sum()) == len(range(0, n, 7))
    newest = a.consumer_observation()[:, -3:].float()
    rgb = a.observe()[1]["rgb"].permute(0, 3, 1, 2).float() / 255
    st = torch.as_tensor(s, device="cuda")
    assert torch.equal(newest[st], rgb[st].half().float()), "the restored envs' newest consumer frame"
    others = torch.as_tensor(np.setdiff1d(np.arange(n), s), device="cuda")
    assert torch.equal(a.consumer_observation()[others], stack[others])
    served0 = a.level_lookahead_info()["served"]
    for t in range(20, 120):
        a_t = acts[t].copy()
        if t % 25 == 0:
            a_t[:] = -1
        _act(envs, a_t)
        out = _outputs(a)
        _assert_same(out, _outputs(control), np.arange(n), f"step {t}")
        for k in ("rgb", "level_end"):
            assert torch.equal(a.final_outputs()[k], control.final_outputs()[k]), f"step {t}: final {k}"
        assert torch.equal(a.consumer_observation(), control.consumer_observation()), f"step {t}: consumer output"
        assert torch.equal(a.rollout(4)["rgb"], control.rollout(4)["rgb"]), f"step {t}: rollout"
    assert a.get_state() == control.get_state()
    info = a.level_lookahead_info()
    assert info["served"] > served0 and info["generated"] > 0, info
    for env in envs + [donor]:
        assert env.errors() == 0
        env.close()


def test_graph_captured_handle(product_lib):
    """set_state after graph replays is ordered behind them (the handle then matches an eager control that restored the
    same blobs after the same steps), and set_state inside a capture raises"""
    import torch

    n = 1024
    kw = dict(distribution_mode="hard", rand_seed=0, **KW)
    g_env, control = _env(n, "coinrun", **kw), _env(n, "coinrun", **kw)
    donor = _env(n, "coinrun", distribution_mode="hard", rand_seed=4, **KW)
    blobs = donor.get_state()
    acts = torch.as_tensor(mt19937_actions(0, n, 60), device="cuda")
    a = torch.zeros(n, dtype=torch.int32, device="cuda")
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        g_env.act(a)
    s = np.random.RandomState(3).permutation(n)[:300]
    for t in range(30):
        a.copy_(acts[t])
        g.replay()
        control.act(acts[t])
    g_env.set_state([blobs[e] for e in s], envs=s)
    control.set_state([blobs[e] for e in s], envs=s)
    _assert_same(_outputs(g_env), _outputs(control), np.arange(n), "after set_state")
    assert g_env.get_state() == control.get_state()
    for t in range(30, 60):
        a.copy_(acts[t])
        g.replay()
        control.act(acts[t])
        _assert_same(_outputs(g_env), _outputs(control), np.arange(n), f"step {t}")
    g2 = torch.cuda.CUDAGraph()
    with pytest.raises(RuntimeError, match="set_state"):
        with torch.cuda.graph(g2):
            g_env.set_state(blobs[:1], envs=[0])
    for env in (g_env, control, donor):
        assert env.errors() == 0
        env.close()


def test_host_buffer_handle(product_lib):
    """observe() after set_state returns the restored frames"""
    n = 256
    donor = _env(n, "caveflyer", distribution_mode="hard", rand_seed=4, **KW)
    for t, a in enumerate(mt19937_actions(0, n, 20)):
        _act([donor], a)
    blobs = donor.get_state()
    want = _outputs(donor)
    host = _env(n, "caveflyer", distribution_mode="hard", rand_seed=0, host_buffers=True, **KW)
    for a in mt19937_actions(1, n, 5):
        host.act(a)
    host.observe()
    s = np.arange(0, n, 3)
    host.set_state([blobs[e] for e in s], envs=s)
    _assert_same(_outputs(host), want, s, "after set_state")
    assert host.get_state(s) == [blobs[e] for e in s]
    assert host.errors() == 0 and donor.errors() == 0
    host.close()
    donor.close()
