"""Per-env level-seed overrides (pgb200_get_next_level_seeds) on the GPU.

The cases of test_level_seeds_on_cpu.py against the oracle's records (emulate_step, level_seed_oracle.py, builds
every override step out of the reference's own plain steps and state blobs), and at benchmark size through the
device-resident Python API: 65 536 envs, overrides refilled by torch every step for a seeded subset of envs,
envs spread over every launch chunk followed by a 64-env oracle, and every env that never gets an override
equal to an untouched control handle. Also the host-buffer path with the Python accessor and an override reset
under the consumer epilogue."""
import ctypes as C

import numpy as np
import pytest

from helpers import make_checked_pair, read_lib_array, run_lockstep
from level_seed_oracle import (check_consumed_kept_and_set_state, emulate_step, refill_plan, run_override_lockstep,
                               use_level_seed_records)
from oracle.record import STANDIN_PACK, oracle_env
from oracle.ref_env import MAX_STATE_SIZE, mt19937_actions

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True, scope="module")
def _level_seed_records():
    """This file's oracle records live in tests/golden/level_seed_records.json.gz."""
    use_level_seed_records()
ALL16 = "bigfish,bossfight,caveflyer,chaser,climber,coinrun,dodgeball,fruitbot,heist,jumper,leaper,maze,miner,ninja,plunder,starpilot"
KW = dict(distribution_mode="hard", num_levels=200, start_level=0, rand_seed=0)
SIXTEEN_64 = "test_gpu_parity.py::test_sixteen_game_list_bit_exact#0"

FORCED = {
    3: ({0: 1000, 1: 1001, 2: 5, 5: 123456}, [0, 1, 2, 5, 9]),
    4: ({1: 2002}, [1]),
    5: ({1: 3003}, [1]),
    30: ({7: 77, 8: 2 ** 31 - 1, 15: 0}, [7, 8, 15, 14]),
    31: ({7: 78}, [7, 14]),
    60: ({e: 500 + e for e in range(16)}, list(range(0, 16, 2))),
}


def forced_plan(t, actions, pending):
    new, force = FORCED.get(t, ({}, []))
    actions[force] = -1
    return new


def test_forced_resets_onto_chosen_seeds(product_lib):
    ref, dut = make_checked_pair(product_lib, 16, "coinrun", **KW)
    assert run_override_lockstep(ref, dut, 61 + 150, forced_plan) >= 18
    ref.close()
    dut.close()


def test_sixteen_game_list_overrides(product_lib):
    ref, dut = make_checked_pair(product_lib, 32, ALL16, **KW)
    assert run_override_lockstep(ref, dut, 300, refill_plan(32, 1)) >= 32 * 300 // 10
    ref.close()
    dut.close()


@pytest.mark.parametrize("name,n,extra,plan_kw,launch_shape", [
    ("maze", 8, dict(use_sequential_levels=True, num_levels=3), dict(low=0, high=50, force_every=16), None),
    ("coinrun", 8, dict(num_levels=1, start_level=5), dict(low=10 ** 6, high=2 ** 31 - 1), None),
    ("coinrun", 8, dict(center_agent=False), {}, None),
    (ALL16, 32, {}, {}, (3, False)),
    ("coinrun", 64, {}, dict(force_every=4), (64, False)),
])
def test_override_options(product_lib, name, n, extra, plan_kw, launch_shape):
    kw = dict(KW)
    kw.update(extra)
    ref, dut = make_checked_pair(product_lib, n, name, launch_shape=launch_shape, **kw)
    assert run_override_lockstep(ref, dut, 200, refill_plan(n, 2, **plan_kw)) > 0
    ref.close()
    dut.close()


def test_array_requested_but_unused_changes_nothing(product_lib):
    """The array exists but is never written: the 16-game run in 3 chunks replays the plain run's record."""
    from level_seed_oracle import next_level_seeds

    ref, dut = make_checked_pair(product_lib, 64, ALL16, key=SIXTEEN_64, launch_shape=(3, False), distribution_mode="hard",
                                 num_levels=200, start_level=0, rand_seed=0)
    seeds = next_level_seeds(dut)
    run_lockstep(ref, dut, 500)
    assert (read_lib_array(seeds) == -1).all()
    ref.close()
    dut.close()


def test_entries_consumed_kept_and_untouched_by_set_state(product_lib):
    check_consumed_kept_and_set_state(product_lib, STANDIN_PACK)


# ------------------------------------------------------------------ benchmark size, device-resident
@pytest.mark.parametrize("name,mode", [("coinrun", "easy"), ("bigfish,coinrun", "hard")])
def test_overrides_at_size(product_lib, name, mode):
    """65 536 envs (8 launch chunks per game). Every step torch refills the consumed overrides of a seeded half
    of the envs, and one action in 16 is -1. Each step: an env that starts an episode with an override pending
    reports it as info level_seed and its entry reads -1, every other entry keeps its value; the envs that never
    get an override equal an untouched control handle; 64 envs from all over the array, exported into a 64-env
    oracle, follow emulate_step of that oracle."""
    import torch

    from procgen_b200 import ProcgenGym3Env

    n_big, n_pick, warm, steps = 65536, 64, 20, 300
    n_games = len(name.split(","))
    rs = np.random.RandomState(17)
    picks = []
    for j in range(n_pick):   # pick j plays game j % n_games, one pick per 1/64 of the array
        lo, hi = j * (n_big // n_pick), (j + 1) * (n_big // n_pick)
        e = int(rs.randint(lo, hi))
        e = e - (e % n_games) + (j % n_games)
        if e >= hi:
            e -= n_games
        picks.append(e)
    picks = np.array(picks)
    pick_t = torch.as_tensor(picks, device="cuda")
    kw = dict(distribution_mode=mode, num_levels=0, start_level=0, rand_seed=0, resource_root=STANDIN_PACK)
    env = ProcgenGym3Env(n_big, name, **kw)
    ctl = ProcgenGym3Env(n_big, name, **kw)
    gen = torch.Generator(device="cuda").manual_seed(21)
    acts = torch.randint(0, 15, (warm + steps, n_big), device="cuda", dtype=torch.int32, generator=gen)
    acts[torch.rand((warm + steps, n_big), device="cuda", generator=gen) < 1 / 16] = -1
    subset = torch.rand(n_big, device="cuda", generator=gen) < 0.5
    with_ovr = torch.as_tensor(np.arange(n_pick) % 4 < 2, device="cuda")   # half of the followed envs (both games) take overrides
    subset[pick_t[with_ovr]] = True
    subset[pick_t[~with_ovr]] = False
    others = ~subset
    seeds = env.next_level_seeds()
    assert bool((seeds == -1).all())
    for t in range(warm):
        env.act(acts[t])
        ctl.act(acts[t])
    env.observe()
    buf = C.create_string_buffer(MAX_STATE_SIZE)

    def blob(e):
        nbytes = int(env._lib.get_state(env._h, int(e), buf, MAX_STATE_SIZE))
        return bytes(buf.raw[:nbytes])

    ref = oracle_env(n_pick, name, product_lib, distribution_mode=mode, num_levels=0, start_level=0, rand_seed=99)
    for j, e in enumerate(picks):
        ref.set_state(j, blob(e))
    ref.observe()
    taken_big = taken_pick = 0
    for t in range(warm, warm + steps):
        fill = subset & (seeds < 0)
        fresh = torch.randint(0, 2 ** 31 - 1, (n_big,), device="cuda", dtype=torch.int32, generator=gen)
        seeds.copy_(torch.where(fill, fresh, seeds))
        pending = seeds.clone()
        pend_pick = pending[pick_t].cpu().numpy()
        pre, took = emulate_step(ref, acts[t][pick_t].cpu().numpy(), pend_pick)
        if t % 50 == 0:
            for j, e in enumerate(picks):
                assert blob(e) == pre[j], f"step {t} env {e}: state blob before the step"
        env.act(acts[t])
        ctl.act(acts[t])
        rew, ob, first = env.observe()
        crew, cob, cfirst = ctl.observe()
        lvl = env.get_info_tensors()["level_seed"]
        took_mask = first & (pending >= 0)
        assert torch.equal(lvl[took_mask], pending[took_mask]), f"step {t}: an override was not played"
        assert torch.equal(seeds, torch.where(took_mask, torch.full_like(pending, -1), pending)), f"step {t}: override array"
        assert torch.equal(ob["rgb"][others], cob["rgb"][others]), f"step {t}: rgb of an env without overrides"
        assert torch.equal(rew[others], crew[others]) and torch.equal(first[others], cfirst[others]), f"step {t}"
        assert torch.equal(lvl[others], ctl.get_info_tensors()["level_seed"][others]), f"step {t}: level_seed"
        r, o, f = ref.observe()
        assert np.array_equal(rew[pick_t].cpu().numpy(), r) and np.array_equal(first[pick_t].cpu().numpy(), f.astype(bool)), f"step {t}"
        assert np.array_equal(ob["rgb"][pick_t].cpu().numpy(), o["rgb"]), f"step {t}: rgb of the followed envs"
        assert np.array_equal(lvl[pick_t].cpu().numpy(), ref.info["level_seed"]), f"step {t}: level_seed of the followed envs"
        taken_big += int(took_mask.sum())
        taken_pick += len(took)
    for j, e in enumerate(picks):
        assert blob(e) == ref.get_state(j), f"state blob of env {e} at the end"
    assert taken_pick > 0 and taken_big > n_big // 4
    assert env.errors() == 0 and ctl.errors() == 0
    for h in (env, ctl, ref):
        h.close()


# ------------------------------------------------------------------ Python API: host buffers, consumer epilogue
def test_host_buffers_python_accessor(product_lib):
    """host_buffers=True: overrides written with torch ops and no synchronisation of the caller's; act() waits
    for the current torch stream before libenv_act."""
    import torch

    from procgen_b200 import ProcgenGym3Env

    n, steps = 64, 200
    env = ProcgenGym3Env(n, "coinrun", host_buffers=True, resource_root=STANDIN_PACK, **KW)
    ref = oracle_env(n, "coinrun", product_lib, **KW)
    seeds = env.next_level_seeds()
    plan = refill_plan(n, 3)
    acts = mt19937_actions(0, n, steps)
    pending = np.full(n, -1, np.int64)
    for t in range(steps):
        a = acts[t].copy()
        for e, s in plan(t, a, pending.copy()).items():
            pending[e] = s
        pre, took = emulate_step(ref, a, pending)
        staged = torch.as_tensor(pending.astype(np.int32)).pin_memory().to("cuda", non_blocking=True)
        seeds.copy_(staged)
        env.act(a)
        rew, ob, first = env.observe()
        r, o, f = ref.observe()
        assert np.array_equal(rew, r) and np.array_equal(first, f), f"step {t}"
        assert np.array_equal(ob["rgb"], o["rgb"]), f"step {t}: rgb"
        for k in ("prev_level_seed", "prev_level_complete", "level_seed"):
            assert np.array_equal(env._info[k], ref.info[k]), f"step {t}: info[{k}]"
        pending[took] = -1
        assert np.array_equal(read_lib_array(seeds), pending), f"step {t}: override array"
    assert env.errors() == 0
    env.close()
    ref.close()


def test_override_reset_under_consumer_epilogue(product_lib):
    """An env that starts the chosen level gets the older frames of its stack zeroed like any episode start."""
    import torch

    from procgen_b200 import ProcgenGym3Env

    n, k = 64, 4
    env = ProcgenGym3Env(n, "coinrun", distribution_mode="easy", num_levels=0, start_level=0, rand_seed=2, resource_root=STANDIN_PACK)
    env.enable_consumer_output(dtype=torch.float16, frames=k)
    seeds = env.next_level_seeds()
    gen = torch.Generator(device="cuda").manual_seed(3)
    for t in range(12):
        env.act(torch.randint(0, 15, (n,), device="cuda", dtype=torch.int32, generator=gen))
    seeds[:32] = torch.arange(1000, 1032, device="cuda", dtype=torch.int32)
    act = torch.full((n,), 4, device="cuda", dtype=torch.int32)
    act[:16] = -1
    env.act(act)
    rew, ob, first = env.observe()
    lvl = env.get_info_tensors()["level_seed"]
    assert bool(first[:16].all())
    assert torch.equal(lvl[:16], torch.arange(1000, 1016, device="cuda", dtype=torch.int32))
    assert bool((seeds[:16] == -1).all())
    untaken = ~first[16:32]
    assert torch.equal(seeds[16:32][untaken], torch.arange(1016, 1032, device="cuda", dtype=torch.int32)[untaken])
    stack = env.consumer_observation().view(n, k, 3, 64, 64)
    newest = (ob["rgb"].permute(0, 3, 1, 2).to(torch.float32) / 255.0).to(torch.float16)
    assert torch.equal(stack[:, -1], newest)
    assert bool((stack[:16, :-1] == 0).all()), "older frames of an override reset not zeroed"
    assert bool((stack[40:][~first[40:]][:, :-1] != 0).any()), "envs that did not reset keep their older frames"
    assert env.errors() == 0
    env.close()
