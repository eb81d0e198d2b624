"""Snapshot slots (env.snapshots() / env.apply_snapshots()) on the GPU, device build only.

A loaded env must continue exactly as its source would have, and an apply must touch nothing but the envs it loads.
Every control here is exact, so no oracle is involved: a handle replaying its own saved states against a twin that
never saved, a handle that loaded slots against a twin that received the same states through set_state, a CUDA graph
against the same calls made eagerly, and a host-buffer handle against its own earlier observation."""
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
    """{name: tensor} of rew, rgb, first and the infos (host arrays for a host-buffer handle)"""
    rew, ob, first = env.observe()
    out = {"rew": rew, "rgb": ob["rgb"], "first": first}
    if env._host_buffers:
        out.update(env._info)
        return {k: np.array(v) for k, v in out.items()}
    out.update(env.get_info_tensors())
    return {k: v.clone() for k, v in out.items()}


def _assert_same(a, b, when, envs=None):
    import torch

    for k in a:
        x, y = (a[k], b[k]) if envs is None else (a[k][envs], b[k][envs])
        if not torch.equal(x, y):
            bad = torch.nonzero((x != y).reshape(len(x), -1).any(1)).flatten()[:8].cpu().numpy()
            raise AssertionError(f"{when}: {k} differs at {'env' if envs is None else 'listed env'} indices {bad}")


def _act(envs, a):
    import torch

    t = torch.as_tensor(a, device="cuda")
    for env in envs:
        env.act(t)


def test_replay_from_saved_states_coinrun_65536(product_lib):
    """Every env saved at t = 20, 64 steps played, every slot loaded back into its env: replaying the same actions then
    gives the outputs of a twin that never left t = 20, byte for byte, at every step. So a slot holds everything a step
    reads."""
    import torch

    n = 65536
    a = _env(n, "coinrun", distribution_mode="easy", rand_seed=0, **KW)
    twin = _env(n, "coinrun", distribution_mode="easy", rand_seed=0, **KW)
    warm, play = mt19937_actions(0, n, 20), mt19937_actions(1, n, 64)
    for t in range(20):
        _act([a, twin], warm[t])
    st = a.snapshots(n)
    everyone = torch.arange(n, dtype=torch.int32, device="cuda")
    st["save_from"].copy_(everyone)
    a.apply_snapshots()
    assert torch.equal(st["source"], everyone) and bool((st["save_from"] == -1).all())
    for t in range(64):
        _act([a], play[t])
    st["load_from"].copy_(everyone)
    a.apply_snapshots()
    assert bool((st["load_from"] == -1).all())
    _assert_same(_outputs(a), _outputs(twin), "after the loads")
    for t in range(64):
        _act([a, twin], play[t])
        _assert_same(_outputs(a), _outputs(twin), f"replayed step {t}")
    assert a.errors() == 0 and twin.errors() == 0
    sample = list(range(0, n, 97))
    assert a.get_state(sample) == twin.get_state(sample)
    a.close()
    twin.close()


@pytest.mark.parametrize("name,mode,n,extra,share", [
    ("coinrun", "easy", 65536, {}, 1.0),
    (ALL16, "hard", 32768, {}, 0.5),
    ("coinrun", "hard", 4096, {"center_agent": False}, 0.5)],
    ids=["coinrun-65536-whole", "all16-32768-half", "coinrun-world-4096-half"])
def test_clones_against_set_state(product_lib, name, mode, n, extra, share):
    """A random set of envs (all of them, or half) saved into slots; ten steps later envs load random slots (in the
    list, about 15 of 16 of them from another game, which must be refused and left as written). The loaded envs must
    hold their sources' save-time blobs, and the handle then runs in lockstep with a twin that received those blobs
    through set_state."""
    import torch

    rng = np.random.RandomState(11)
    games = 16 if name == ALL16 else 1
    kw = dict(distribution_mode=mode, rand_seed=0, **KW, **extra)
    a, twin = _env(n, name, **kw), _env(n, name, **kw)
    acts = mt19937_actions(2, n, 70)
    for t in range(20):
        _act([a, twin], acts[t])
    slots = int(n * share)
    st = a.snapshots(slots)
    sources = rng.permutation(n)[:slots]
    blobs = a.get_state(sources)
    st["save_from"].copy_(torch.as_tensor(sources, dtype=torch.int32))
    a.apply_snapshots()
    assert np.array_equal(st["source"].cpu().numpy(), sources)
    for t in range(20, 30):
        _act([a, twin], acts[t])
    targets = rng.permutation(n)[:slots]
    picks = rng.randint(0, slots, size=slots)
    load = np.full(n, -1, np.int32)
    load[targets] = picks
    st["load_from"].copy_(torch.as_tensor(load))
    a.apply_snapshots()
    ok = sources[picks] % games == targets % games
    assert ok.all() or (games > 1 and 0 < ok.sum() < slots)
    left = st["load_from"].cpu().numpy()
    assert (left[targets[ok]] == -1).all() and np.array_equal(left[targets[~ok]], picks[~ok]), "refused entries"
    loaded = targets[ok]
    want = [blobs[p] for p in picks[ok]]
    assert a.get_state(loaded[:4096]) == want[:4096]
    twin.set_state(want, envs=loaded)
    _assert_same(_outputs(a), _outputs(twin), "after the loads")
    for t in range(30, 70):
        _act([a, twin], acts[t])
        _assert_same(_outputs(a), _outputs(twin), f"step {t}")
    sample = list(range(0, n, 13))
    assert a.get_state(sample) == twin.get_state(sample)
    assert a.errors() == 0 and twin.errors() == 0
    a.close()
    twin.close()


def test_every_opt_in(product_lib):
    """Final outputs, the pause mask, the rollout, a 4-frame consumer output and level lookahead on: an apply leaves the
    rollout, the final outputs and the mask alone, rewrites the loaded envs' newest consumer frame and no other, and the
    handle then runs in lockstep with a control without lookahead (which changes no output) that received the same
    states through set_state, through resets forced with action -1."""
    import torch

    n, name = 2048, "coinrun"
    rng = np.random.RandomState(1)
    kw = dict(distribution_mode="hard", rand_seed=0, **KW)
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
    st = a.snapshots(n // 4)
    sources = rng.permutation(n)[: n // 4]
    blobs = a.get_state(sources)
    st["save_from"].copy_(torch.as_tensor(sources, dtype=torch.int32))
    a.apply_snapshots()
    for t in range(20, 30):
        _act(envs, acts[t])
    targets = rng.permutation(n)[: n // 3]
    picks = rng.randint(0, n // 4, size=len(targets))
    torch.cuda.synchronize()
    before = {k: v.clone() for k, v in a.rollout(4).items()}
    final = {k: v.clone() for k, v in a.final_outputs().items()}
    stack = a.consumer_observation().clone()
    st["load_from"][torch.as_tensor(targets, device="cuda")] = torch.as_tensor(picks, dtype=torch.int32, device="cuda")
    a.apply_snapshots()
    control.set_state([blobs[p] for p in picks], envs=targets)
    torch.cuda.synchronize()
    assert bool((st["load_from"] == -1).all())
    for k, v in a.rollout(4).items():
        assert torch.equal(v, before[k]), f"apply changed the rollout's {k}"
    for k, v in a.final_outputs().items():
        assert torch.equal(v, final[k]), f"apply changed the final outputs' {k}"
    assert int(a.pause_mask().sum()) == len(range(0, n, 7))
    newest = a.consumer_observation()[:, -3:].float()
    rgb = a.observe()[1]["rgb"].permute(0, 3, 1, 2).float() / 255
    tt = torch.as_tensor(targets, device="cuda")
    assert torch.equal(newest[tt], rgb[tt].half().float()), "the loaded envs' newest consumer frame"
    others = torch.as_tensor(np.setdiff1d(np.arange(n), targets), device="cuda")
    assert torch.equal(a.consumer_observation()[others], stack[others])
    _assert_same(_outputs(a), _outputs(control), "after the loads")
    served0 = a.level_lookahead_info()["served"]
    for t in range(30, 120):
        a_t = acts[t].copy()
        if t % 25 == 0:
            a_t[:] = -1
        _act(envs, a_t)
        _assert_same(_outputs(a), _outputs(control), f"step {t}")
        for k in ("rgb", "level_end"):
            assert torch.equal(a.final_outputs()[k], control.final_outputs()[k]), f"step {t}: final {k}"
        assert torch.equal(a.consumer_observation(), control.consumer_observation()), f"step {t}: consumer output"
        assert torch.equal(a.rollout(4)["rgb"], control.rollout(4)["rgb"]), f"step {t}: rollout"
    assert a.get_state() == control.get_state()
    info = a.level_lookahead_info()
    assert info["served"] > served0 and info["generated"] > 0, info
    for env in envs:
        assert env.errors() == 0
        env.close()


def test_graph_capture(product_lib):
    """An 8-step CUDA graph of [torch refills save_from and load_from, apply_snapshots(), act()] replayed twice against
    the same calls made eagerly on a twin; and the first snapshots() call raises inside a capture."""
    import torch

    n, slots, steps = 4096, 64, 8
    kw = dict(distribution_mode="hard", rand_seed=0, **KW)
    g_env, eager = _env(n, "coinrun", **kw), _env(n, "coinrun", **kw)
    for t, acts in enumerate(mt19937_actions(0, n, 10)):
        _act([g_env, eager], acts)
    stores = [g_env.snapshots(slots), eager.snapshots(slots)]
    rng = np.random.RandomState(5)

    def plan():
        """per step: (save_from, load_from, actions); half the slots save, 1 % of the envs load, at first also from slots
        still empty"""
        out = []
        for _ in range(steps):
            save = np.where(rng.rand(slots) < 0.5, rng.randint(0, n, size=slots), -1).astype(np.int32)
            load = np.full(n, -1, np.int32)
            load[rng.permutation(n)[: n // 100]] = rng.randint(0, slots, size=n // 100)
            out.append((save, load, rng.randint(0, 15, size=n).astype(np.int32)))
        return [tuple(torch.as_tensor(x, device="cuda") for x in step) for step in out]

    inputs = [[torch.empty_like(x) for x in step] for step in plan()]
    a = torch.zeros(n, dtype=torch.int32, device="cuda")
    for env in (g_env, eager):  # every kernel is loaded before the capture; with every entry -1 an apply changes nothing
        env.apply_snapshots()
        env.act(a)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for save, load, act in inputs:
            stores[0]["save_from"].copy_(save)
            stores[0]["load_from"].copy_(load)
            g_env.apply_snapshots()
            g_env.act(act)
    for replay in range(2):
        p = plan()
        for dst, src in zip(inputs, p):
            for d, s in zip(dst, src):
                d.copy_(s)
        g.replay()
        for save, load, act in p:
            stores[1]["save_from"].copy_(save)
            stores[1]["load_from"].copy_(load)
            eager.apply_snapshots()
            eager.act(act)
        _assert_same(_outputs(g_env), _outputs(eager), f"replay {replay}")
        for k in ("save_from", "load_from", "source"):
            assert torch.equal(stores[0][k], stores[1][k]), f"replay {replay}: {k}"
        assert g_env.get_state() == eager.get_state(), f"replay {replay}: blobs differ"
    assert int((stores[1]["source"] >= 0).sum()) > 0
    fresh = _env(256, "coinrun", **kw)
    g2 = torch.cuda.CUDAGraph()
    with pytest.raises(RuntimeError, match="snapshots"):
        with torch.cuda.graph(g2):
            fresh.snapshots(4)
    for env in (g_env, eager, fresh):
        assert env.errors() == 0
        env.close()


def test_host_buffer_handle(product_lib):
    """On a host-buffer handle, observe() after an apply returns the loaded envs' frames: those the handle showed when
    their states were saved"""
    n = 256
    host = _env(n, "caveflyer", distribution_mode="hard", rand_seed=0, host_buffers=True, **KW)
    for a in mt19937_actions(1, n, 5):
        host.act(a)
    want = _outputs(host)
    st = host.snapshots(n)
    st["save_from"][:] = st["save_from"].new_tensor(np.arange(n, dtype=np.int32))
    host.apply_snapshots()
    for a in mt19937_actions(2, n, 5):
        host.act(a)
    host.observe()
    envs = np.arange(0, n, 3)
    load = np.full(n, -1, np.int32)
    load[envs] = envs
    st["load_from"].copy_(st["load_from"].new_tensor(load))
    host.apply_snapshots()
    got = _outputs(host)
    for k in want:
        assert np.array_equal(got[k][envs], want[k][envs]), f"{k} after the loads"
    assert int((st["load_from"] >= 0).sum()) == 0
    assert host.errors() == 0
    host.close()


def test_close_returns_device_memory(product_lib):
    """Three handles, each with a store of about 1.3 GB that saves and loads, leave the device's free memory where it was"""
    import torch

    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    for _ in range(3):
        env = _env(1024, "coinrun", distribution_mode="easy", rand_seed=0, **KW)
        st = env.snapshots(16384)
        st["save_from"][:1024] = torch.arange(1024, dtype=torch.int32, device="cuda")
        st["load_from"].copy_(torch.arange(1024, dtype=torch.int32, device="cuda").flip(0))
        env.apply_snapshots()
        env.act(torch.zeros(1024, dtype=torch.int32, device="cuda"))
        env.close()
        del env, st
    torch.cuda.synchronize()
    free1 = torch.cuda.mem_get_info()[0]
    assert free1 >= free0 - (256 << 20), f"{(free0 - free1) >> 20} MiB not returned"
