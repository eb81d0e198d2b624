"""The pause mask (pgb200_get_pause_mask) on the GPU.

The emulated cases of test_pause_on_cpu.py against the oracle's records (tests/golden/pause_records.json.gz), and at
benchmark size through the device-resident Python API: a time-shift check at 65 536 envs (pausing is a pure delay,
so a paused handle equals a control handle that never pauses, each env shifted by its own paused steps), the
consumer ring of a paused env, a CUDA graph with the mask refilled inside it, and host-buffer mode."""
import ctypes as C

import numpy as np
import pytest

from final_obs_oracle import final_oracle_env, near_timeout
from helpers import make_checked_pair
from level_seed_oracle import refill_plan
from oracle.record import STANDIN_PACK
from oracle.ref_env import MAX_STATE_SIZE, RefVecEnv
from pause_oracle import (all_plan, check_set_state_into_paused_env, episode_end_plan, halves_plan, long_plan,
                          run_pause_lockstep, use_pause_records, zero_plan)

pytestmark = pytest.mark.gpu

ALL16 = "bigfish,bossfight,caveflyer,chaser,climber,coinrun,dodgeball,fruitbot,heist,jumper,leaper,maze,miner,ninja,plunder,starpilot"
KW = dict(distribution_mode="hard", num_levels=200, start_level=0, rand_seed=0)


@pytest.fixture(autouse=True, scope="module")
def _pause_records():
    use_pause_records()


def _close(*envs):
    for e in envs:
        e.close()


# ------------------------------------------------------------------ against the oracle's records
@pytest.mark.parametrize("mode", ["easy", "hard"])
def test_sixteen_games_random_halves(product_lib, mode):
    ref, dut = make_checked_pair(product_lib, 32, ALL16, **dict(KW, distribution_mode=mode))
    run_pause_lockstep(ref, dut, 100, halves_plan(32, 1), blob_every=5)
    _close(ref, dut)


def test_long_pauses_span_the_time_limit(product_lib):
    n = 32
    ref, dut = make_checked_pair(product_lib, n, ALL16, **KW)
    near_timeout([ref, dut], n)
    assert run_pause_lockstep(ref, dut, 80, long_plan(n, 3), blob_every=5).sum(0).min() >= 20
    _close(ref, dut)


def test_pause_at_episode_end(product_lib):
    n = 32
    ref, dut = make_checked_pair(product_lib, n, ALL16, **KW)
    near_timeout([ref, dut], n, steps_left=40)
    assert run_pause_lockstep(ref, dut, 60, episode_end_plan(n), blob_every=5)[-1].all()
    _close(ref, dut)


def test_every_env_paused_and_zero_mask(product_lib):
    ref, dut = make_checked_pair(product_lib, 16, ALL16, **KW)
    run_pause_lockstep(ref, dut, 50, all_plan(16), blob_every=5)
    _close(ref, dut)
    ref, dut = make_checked_pair(product_lib, 16, ALL16, **KW)
    run_pause_lockstep(ref, dut, 50, zero_plan(16), blob_every=10)
    _close(ref, dut)


def test_sequential_levels(product_lib):
    kw = dict(distribution_mode="easy", num_levels=3, start_level=0, rand_seed=0, use_sequential_levels=True)
    ref, dut = make_checked_pair(product_lib, 8, "maze", **kw)
    run_pause_lockstep(ref, dut, 200, halves_plan(8, 4), blob_every=5)
    _close(ref, dut)


@pytest.mark.parametrize("name", ["coinrun", "climber", "caveflyer", "ninja", "jumper"])
def test_whole_world_view(product_lib, name):
    ref, dut = make_checked_pair(product_lib, 8, name, **dict(KW, center_agent=False))
    run_pause_lockstep(ref, dut, 60, halves_plan(8, 5), blob_every=5)
    _close(ref, dut)


def test_overrides_refilled_every_step(product_lib):
    ref, dut = make_checked_pair(product_lib, 32, ALL16, **KW)
    run_pause_lockstep(ref, dut, 100, halves_plan(32, 6), plan=refill_plan(32, 1, force_every=4), overrides=True, blob_every=5)
    _close(ref, dut)


def test_final_outputs(product_lib):
    n = 32
    ref, fin = final_oracle_env(n, ALL16, product_lib, **KW)
    dut = RefVecEnv(n, ALL16, lib_path=product_lib, resource_root=STANDIN_PACK, **KW)
    rs = np.random.RandomState(7)

    def plan(t, actions, pending):
        actions[rs.randint(16, size=n) == 0] = -1
        return {}

    run_pause_lockstep(ref, dut, 100, episode_end_plan(n, release_every=20), plan=plan, final=fin, blob_every=5)
    _close(ref, fin, dut)


@pytest.mark.parametrize("chunks", [3, 64])
def test_forced_launch_shapes(product_lib, chunks):
    n = 48 if chunks == 3 else 32
    ref, dut = make_checked_pair(product_lib, n, ALL16, launch_shape=(chunks, False), **KW)
    run_pause_lockstep(ref, dut, 60, halves_plan(n, 8), blob_every=5)
    _close(ref, dut)


def test_action_minus_one_on_paused_envs(product_lib):
    ref, dut = make_checked_pair(product_lib, 16, ALL16, **KW)
    run_pause_lockstep(ref, dut, 60, halves_plan(16, 9), force_paused=True, blob_every=5)
    _close(ref, dut)


def test_set_state_into_paused_env(product_lib):
    kw = dict(KW, lib_path=product_lib, resource_root=STANDIN_PACK)
    dut = RefVecEnv(8, "coinrun", **kw)
    donor = RefVecEnv(8, "coinrun", **dict(kw, rand_seed=7))
    check_set_state_into_paused_env(donor, dut)
    _close(dut, donor)


# ------------------------------------------------------------------ benchmark size, device-resident
def _actions(torch, n_steps, num):
    """Env e's action at its own step n: a fixed function of (e, n), -1 about once in 16."""
    e = torch.arange(num, device="cuda", dtype=torch.int64)
    h = (e * 2654435761 + n_steps * 40503 + 12345) % 1000003
    return (h % 16 - 1).to(torch.int32)


@pytest.mark.parametrize("name,mode", [("coinrun", "easy"), ("bigfish", "hard"), (ALL16, "hard")])
def test_pause_is_a_time_shift(product_lib, name, mode):
    """65 536 envs (8 launch chunks per game; the 16-game list has a pause in every launch). Env e's action is a
    fixed function of (e, n_e), n_e = the steps env e has actually taken. A handle under random multi-step pauses
    then equals a control handle that never pauses, shifted per env: when the control reaches step t, rgb, infos
    and first of the envs with final n_e = t are snapshotted, and compared at the end with the paused handle's
    (first and rew only where the last step did not pause the env), as are the state blobs of 256 envs spread over
    all 8 chunks."""
    import torch

    from procgen_b200 import ProcgenGym3Env

    n, steps = 65536, 160
    kw = dict(distribution_mode=mode, num_levels=0, start_level=0, rand_seed=0, resource_root=STANDIN_PACK)
    env = ProcgenGym3Env(n, name, **kw)
    mask = env.pause_mask()
    gen = torch.Generator(device="cuda").manual_seed(3)
    count = torch.zeros(n, dtype=torch.int64, device="cuda")
    paused = torch.zeros(n, dtype=torch.bool, device="cuda")
    for t in range(steps):
        # pauses last several steps: a running env pauses with p = 0.25, a paused one resumes with p = 0.3
        u = torch.rand(n, device="cuda", generator=gen)
        paused = torch.where(paused, u >= 0.3, u < 0.25)
        mask.copy_(paused.to(torch.uint8))
        env.act(_actions(torch, count, n))
        count += (~paused).to(torch.int64)
    rew, ob, first = env.observe()
    last_ran = ~paused
    assert bool(paused.any()) and bool(last_ran.any()) and int(count.min()) < int(count.max())
    buf = C.create_string_buffer(MAX_STATE_SIZE)

    def blob(h, e):
        k = int(h._lib.get_state(h._h, int(e), buf, MAX_STATE_SIZE))
        return bytes(buf.raw[:k])

    picks = [int(c * (n // 8) + j * (n // 8 // 32) + (c * 7 + j) % 16) for c in range(8) for j in range(32)]
    want_blob = {e: blob(env, e) for e in picks}
    ctl = ProcgenGym3Env(n, name, **kw)
    snap_rgb = torch.zeros_like(ob["rgb"])
    snap_first = torch.zeros_like(first)
    snap_rew = torch.zeros_like(rew)
    snap_info = {k: torch.zeros_like(v) for k, v in env.get_info_tensors().items()}
    cnt_cpu = count.cpu().numpy()
    for t in range(int(count.max()) + 1):
        if t > 0:
            ctl.act(_actions(torch, torch.full((n,), t - 1, dtype=torch.int64, device="cuda"), n))
        crew, cob, cfirst = ctl.observe()
        sel = (count == t).nonzero().squeeze(1)
        snap_rgb[sel] = cob["rgb"][sel]
        snap_first[sel] = cfirst[sel]
        snap_rew[sel] = crew[sel]
        for k, v in ctl.get_info_tensors().items():
            snap_info[k][sel] = v[sel]
        for e in picks:
            if cnt_cpu[e] == t:
                assert blob(ctl, e) == want_blob[e], f"env {e} after {t} own steps: state blobs differ"
    assert torch.equal(snap_rgb, ob["rgb"]), f"rgb differs at envs {(snap_rgb != ob['rgb']).flatten(1).any(1).nonzero()[:8].tolist()}"
    for k, v in env.get_info_tensors().items():
        assert torch.equal(snap_info[k], v), f"info {k}"
    assert torch.equal(snap_first[last_ran], first[last_ran]) and torch.equal(snap_rew[last_ran], rew[last_ran])
    assert not bool(first[paused].any()) and not bool(rew[paused].any())
    assert env.errors() == 0 and ctl.errors() == 0
    env.close()
    ctl.close()


@pytest.mark.parametrize("k", [1, 4])
@pytest.mark.parametrize("dtype", ["float16", "bfloat16"])
def test_consumer_ring_repeats_a_paused_frame(product_lib, k, dtype):
    """With the consumer output on, a paused env's newest frame is its current rgb again and its older frames are
    kept: the stack equals one built with torch ops from the u8 frames by the usual rule (shift in the current frame;
    zero the older ones where first is set), with a pause in the mix."""
    import torch

    from procgen_b200 import ProcgenGym3Env

    dt = getattr(torch, dtype)
    n = 4096
    kw = dict(distribution_mode="hard", num_levels=0, start_level=0, rand_seed=2, resource_root=STANDIN_PACK)
    env = ProcgenGym3Env(n, "bigfish,coinrun", **kw)
    env.enable_consumer_output(dtype=dt, frames=k)
    mask = env.pause_mask()

    def frame():
        return (env.observe()[1]["rgb"].permute(0, 3, 1, 2).float() / 255.0).to(dt)

    stack = torch.zeros((n, k, 3, 64, 64), dtype=dt, device="cuda")
    stack[:, -1] = frame()
    gen = torch.Generator(device="cuda").manual_seed(8)
    paused = torch.zeros(n, dtype=torch.bool, device="cuda")
    for t in range(120):
        u = torch.rand(n, device="cuda", generator=gen)
        paused = torch.where(paused, u >= 0.2, u < 0.3)
        mask.copy_(paused.to(torch.uint8))
        a = torch.randint(-1, 15, (n,), device="cuda", dtype=torch.int32, generator=gen)
        env.act(a)
        _, _, first = env.observe()
        stack = torch.cat([stack[:, 1:], frame()[:, None]], 1)
        stack[first, :-1] = 0
        got = env.consumer_observation().reshape(n, k, 3, 64, 64)
        assert torch.equal(got, stack), f"step {t}: stacks differ at envs {(got != stack).flatten(1).any(1).nonzero()[:8].tolist()}"
    assert env.errors() == 0
    env.close()


def test_graph_with_the_mask_refilled_inside(product_lib):
    """A graph of 8 act() calls, each behind a copy into the mask, replayed: equal to eager steps with the same masks.
    The first pause_mask() call is refused inside a capture."""
    import torch

    from procgen_b200 import ProcgenGym3Env

    n, reps = 4096, 10
    kw = dict(distribution_mode="hard", num_levels=0, start_level=0, rand_seed=5, resource_root=STANDIN_PACK)
    other = ProcgenGym3Env(64, "coinrun", **kw)
    with pytest.raises(RuntimeError, match="pause_mask"):
        with torch.cuda.graph(torch.cuda.CUDAGraph()):
            other.pause_mask()
    other.close()
    eager = ProcgenGym3Env(n, "bigfish,coinrun", **kw)
    graph = ProcgenGym3Env(n, "bigfish,coinrun", **kw)
    me, mg = eager.pause_mask(), graph.pause_mask()
    gen = torch.Generator(device="cuda").manual_seed(4)
    acts = torch.randint(-1, 15, (reps * 8, n), device="cuda", dtype=torch.int32, generator=gen)
    masks = (torch.rand((reps * 8, n), device="cuda", generator=gen) < 0.5).to(torch.uint8)
    abuf = torch.zeros((8, n), device="cuda", dtype=torch.int32)
    mbuf = torch.zeros((8, n), device="cuda", dtype=torch.uint8)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for s in range(8):
            mg.copy_(mbuf[s])
            graph.act(abuf[s])
    torch.cuda.synchronize()
    for r in range(reps):
        abuf.copy_(acts[8 * r:8 * r + 8])
        mbuf.copy_(masks[8 * r:8 * r + 8])
        g.replay()
        for s in range(8):
            me.copy_(masks[8 * r + s])
            eager.act(acts[8 * r + s])
        re_, oe, fe = eager.observe()
        rg, og, fg = graph.observe()
        assert torch.equal(oe["rgb"], og["rgb"]) and torch.equal(re_, rg) and torch.equal(fe, fg), f"replay {r}"
        for key, v in eager.get_info_tensors().items():
            assert torch.equal(v, graph.get_info_tensors()[key]), f"replay {r}: info {key}"
    assert eager.errors() == 0 and graph.errors() == 0
    eager.close()
    graph.close()


def test_host_buffers_with_the_python_accessor(product_lib):
    """host_buffers=True: pause_mask() written with torch, act() waits for the writes; equal to a device-resident handle."""
    import torch

    from procgen_b200 import ProcgenGym3Env

    n = 256
    kw = dict(distribution_mode="hard", num_levels=0, start_level=0, rand_seed=6, resource_root=STANDIN_PACK)
    host = ProcgenGym3Env(n, "bigfish,coinrun", host_buffers=True, **kw)
    dev = ProcgenGym3Env(n, "bigfish,coinrun", **kw)
    mh, md = host.pause_mask(), dev.pause_mask()
    assert mh.is_cuda and mh.dtype == torch.uint8 and mh.shape == (n,)
    gen = torch.Generator(device="cuda").manual_seed(9)
    for t in range(80):
        m = (torch.rand(n, device="cuda", generator=gen) < 0.5).to(torch.uint8)
        a = torch.randint(-1, 15, (n,), device="cuda", dtype=torch.int32, generator=gen)
        mh.copy_(m)
        md.copy_(m)
        host.act(a.cpu().numpy())
        dev.act(a)
        r1, o1, f1 = host.observe()
        r2, o2, f2 = dev.observe()
        assert np.array_equal(r1, r2.cpu().numpy()) and np.array_equal(f1, f2.cpu().numpy()), f"step {t}"
        assert np.array_equal(o1["rgb"], o2["rgb"].cpu().numpy()), f"step {t}: rgb"
    host.close()
    dev.close()
