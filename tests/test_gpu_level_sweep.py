"""Level generation swept over the seed range on the GPU, against the oracle's records.

Level generation is where the device code departs furthest from the host debug build: the warp-wide MT19937
refill and tempering (pg_rng.cuh), the wall-list and set-relabel steps of pg_mazegen.cuh, the room stamping
of pg_roomgen.cuh, jumper's and caveflyer's cave passes and the chunked erase of pg_engine.cuh all have
branches that only the device compiles. This file puts envs on about a thousand seeds per (game, mode) pair
(edge seeds, the fullest levels of tests/golden/level_extremes.json, uniform draws over [0, 2^31)) through
the per-env override and compares every level byte for byte, right after generation and after a rollout
(level_sweep.py). Records: tests/golden/level_sweep_records.json.gz."""
import ctypes as C

import numpy as np
import pytest

from helpers import make_checked_pair
from level_seed_oracle import emulate_step
from level_sweep import ALL16, LEVEL_SWEEP_RECORDS, PAIRS, WHOLE_WORLD, run_level_sweep, run_sequential_wrap, sweep_seeds
from oracle.record import STANDIN_PACK, oracle_env, use_records
from oracle.ref_env import MAX_STATE_SIZE

pytestmark = pytest.mark.gpu

N_SEEDS, N_ENVS, ROLLOUT = 1024, 256, 24


@pytest.fixture(autouse=True, scope="module")
def _level_sweep_records():
    use_records(LEVEL_SWEEP_RECORDS)


def sweep(lib, name, mode, count, n=N_ENVS, **extra):
    ref, dut = make_checked_pair(lib, n, name, distribution_mode=mode, num_levels=0, start_level=0, rand_seed=0, **extra)
    assert run_level_sweep(ref, dut, sweep_seeds(name, mode, count), ROLLOUT) == -(-count // n)
    ref.close()
    dut.close()


@pytest.mark.parametrize("name,mode", PAIRS)
def test_level_sweep(product_lib, name, mode):
    sweep(product_lib, name, mode, N_SEEDS)


def test_sixteen_game_list_restrict_themes(product_lib):
    """restrict_themes masks the theme for the aspect ratios level logic reads, not only for the sprite."""
    sweep(product_lib, ALL16, "hard", N_SEEDS, restrict_themes=True)


@pytest.mark.parametrize("name,mode", WHOLE_WORLD)
def test_whole_world_view(product_lib, name, mode):
    """center_agent=False: the cell size of the whole-world view follows each level's world size."""
    sweep(product_lib, name, mode, 512, center_agent=False)


def test_sequential_levels_wrap_to_negative_seeds(product_lib):
    ref, dut = make_checked_pair(product_lib, 32, "jumper", distribution_mode="easy", num_levels=0, start_level=0, rand_seed=0,
                                 use_sequential_levels=True)
    assert len(run_sequential_wrap(ref, dut, 800)) > 0, "no env reached a negative level seed"
    ref.close()
    dut.close()


def test_every_chunk_generates_at_once(product_lib):
    """A 65 536-env 16-game handle (8 launch chunks per game) with every env put on a chosen seed in the same
    step. 256 envs from all over the array are exported into a 256-env oracle before that step; they must
    follow emulate_step of the oracle (outputs, then 24 steps, state blobs at the end), every env must report
    its seed and every override must be consumed."""
    import torch

    from procgen_b200 import ProcgenGym3Env

    n_big, n_pick, warm = 65536, 256, 8
    n_games = 16
    rs = np.random.RandomState(31)
    picks = []
    for j in range(n_pick):   # pick j plays game j % 16, one pick per 1/256 of the array
        lo, hi = j * (n_big // n_pick), (j + 1) * (n_big // n_pick)
        e = int(rs.randint(lo, hi))
        e = e - (e % n_games) + (j % n_games)
        if e >= hi:
            e -= n_games
        picks.append(e)
    picks = np.array(picks)
    pick_t = torch.as_tensor(picks, device="cuda")
    kw = dict(distribution_mode="hard", num_levels=0, start_level=0, rand_seed=0)
    env = ProcgenGym3Env(n_big, ALL16, resource_root=STANDIN_PACK, **kw)
    gen = torch.Generator(device="cuda").manual_seed(5)
    for t in range(warm):
        env.act(torch.randint(0, 15, (n_big,), device="cuda", dtype=torch.int32, generator=gen))
    env.observe()
    buf = C.create_string_buffer(MAX_STATE_SIZE)

    def blob(e):
        nbytes = int(env._lib.get_state(env._h, int(e), buf, MAX_STATE_SIZE))
        return bytes(buf.raw[:nbytes])

    ref = oracle_env(n_pick, ALL16, product_lib, **dict(kw, rand_seed=99))
    for j, e in enumerate(picks):
        ref.set_state(j, blob(e))
    ref.observe()
    chosen = np.array(sweep_seeds(ALL16, "hard", n_big), np.int64)
    seeds = env.next_level_seeds()
    seeds.copy_(torch.as_tensor(chosen.astype(np.int32), device="cuda"))
    force = torch.full((n_big,), -1, device="cuda", dtype=torch.int32)
    _, took = emulate_step(ref, np.full(n_pick, -1, np.int32), chosen[picks])
    assert took == list(range(n_pick))
    env.act(force)
    rew, ob, first = env.observe()
    lvl = env.get_info_tensors()["level_seed"].cpu().numpy()
    assert np.array_equal(lvl, chosen), "an env did not play its chosen seed"
    assert bool((seeds == -1).all()) and bool(first.all())
    acts = torch.randint(0, 15, (ROLLOUT + 1, n_big), device="cuda", dtype=torch.int32, generator=gen)
    for t in range(ROLLOUT + 1):
        r, o, f = ref.observe()
        assert np.array_equal(rew[pick_t].cpu().numpy(), r) and np.array_equal(first[pick_t].cpu().numpy(), f.astype(bool)), f"step {t}"
        assert np.array_equal(ob["rgb"][pick_t].cpu().numpy(), o["rgb"]), f"step {t}: rgb of the followed envs"
        info = env.get_info_tensors()
        for k, v in ref.info.items():
            assert np.array_equal(info[k][pick_t].cpu().numpy(), v), f"step {t}: info[{k}] of the followed envs"
        if t == 0:
            for j, e in enumerate(picks):
                assert blob(e) == ref.get_state(j), f"env {e}: state blob of the generated level"
        if t == ROLLOUT:
            break
        env.act(acts[t])
        ref.act(acts[t][pick_t].cpu().numpy())
        rew, ob, first = env.observe()
    for j, e in enumerate(picks):
        assert blob(e) == ref.get_state(j), f"env {e}: state blob after {ROLLOUT} steps"
    assert env.errors() == 0
    env.close()
    ref.close()
