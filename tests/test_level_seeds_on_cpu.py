"""Per-env level-seed overrides (pgb200_get_next_level_seeds) in the host debug build, against the live oracle:
every step of a run with overrides equals the reference's own step with the same level chosen (emulate_step in
level_seed_oracle.py), state blobs included, and the override array is consumed exactly where a reset took it."""
import numpy as np
import pytest

from helpers import make_pair, read_lib_array, run_lockstep, write_lib_array
from level_seed_oracle import (check_consumed_kept_and_set_state, emulate_step, field_offsets, next_level_seeds, patch_fields,
                               refill_plan, run_override_lockstep)
from oracle.state_blob import parse

ALL16 = "bigfish,bossfight,caveflyer,chaser,climber,coinrun,dodgeball,fruitbot,heist,jumper,leaper,maze,miner,ninja,plunder,starpilot"
KW = dict(distribution_mode="hard", num_levels=200, start_level=0, rand_seed=0)

# env -> seed, written before the given step; with the env's action forced to -1 where `force` says so
FORCED = {
    3: ({0: 1000, 1: 1001, 2: 5, 5: 123456}, [0, 1, 2, 5, 9]),   # env 9: action -1 without an override
    4: ({1: 2002}, [1]),                                          # env 1 again, one step later
    5: ({1: 3003}, [1]),                                          # ... and again
    30: ({7: 77, 8: 2 ** 31 - 1, 15: 0}, [7, 8, 15, 14]),
    31: ({7: 78}, [7, 14]),
    60: ({e: 500 + e for e in range(16)}, list(range(0, 16, 2))),  # odd envs keep theirs until a natural end
}


def forced_plan(t, actions, pending):
    new, force = FORCED.get(t, ({}, []))
    actions[force] = -1
    return new


def test_forced_resets_onto_chosen_seeds(ref_lib, hostsim_lib):
    """Overrides fired with action -1 at several steps (twice and three times in a row for some envs, action -1
    without an override for others), then 150 more lockstep steps in which pending overrides meet natural
    episode ends."""
    ref, dut = make_pair(hostsim_lib, 16, "coinrun", **KW)
    taken = run_override_lockstep(ref, dut, 61 + 150, forced_plan)
    assert taken >= 18   # every forced one
    ref.close()
    dut.close()


def test_sixteen_game_list_overrides(ref_lib, hostsim_lib):
    """Every env of the 16-game list has an override pending at all times (refilled when consumed) and one
    action in 8 is -1: natural and forced episode ends in every game take overrides."""
    ref, dut = make_pair(hostsim_lib, 32, ALL16, **KW)
    taken = run_override_lockstep(ref, dut, 300, refill_plan(32, 1))
    assert taken >= 32 * 300 // 10   # about one env-step in 8 is a forced end
    ref.close()
    dut.close()


@pytest.mark.parametrize("name,n,extra,plan_kw,launch_shape", [
    ("maze", 8, dict(use_sequential_levels=True, num_levels=3), dict(low=0, high=50, force_every=16), None),
    ("coinrun", 8, dict(num_levels=1, start_level=5), dict(low=10 ** 6, high=2 ** 31 - 1), None),   # seeds outside the range
    ("coinrun", 8, dict(center_agent=False), {}, None),     # the whole-world instantiation
    (ALL16, 32, {}, {}, (3, False)),                        # joint list in 3 uneven chunks per game
    ("coinrun", 64, {}, dict(force_every=4), (64, False)),  # one env per chunk
])
def test_override_options(ref_lib, hostsim_lib, name, n, extra, plan_kw, launch_shape):
    kw = dict(KW)
    kw.update(extra)
    ref, dut = make_pair(hostsim_lib, n, name, launch_shape=launch_shape, **kw)
    assert run_override_lockstep(ref, dut, 200, refill_plan(n, 2, **plan_kw)) > 0
    ref.close()
    dut.close()


def test_sequential_levels_continue_from_override(ref_lib, hostsim_lib):
    """use_sequential_levels: a level completed after an override was taken is followed by level s + 997."""
    ref, dut = make_pair(hostsim_lib, 8, "maze", distribution_mode="easy", num_levels=3, start_level=0, rand_seed=0,
                         use_sequential_levels=True)
    seeds = next_level_seeds(dut)
    write_lib_array(seeds, np.arange(8) + 4000)
    acts = np.full(8, -1, np.int32)
    pre, took = emulate_step(ref, acts, read_lib_array(seeds))
    dut.act(acts)
    assert took == list(range(8))
    from helpers import assert_same_observation

    from oracle.ref_env import mt19937_actions

    assert_same_observation(ref, dut, 0)
    assert (dut.info["level_seed"] == np.arange(8) + 4000).all()
    # from here on the envs play on; a completed level is followed by s + 997
    followed = np.zeros(8, bool)
    acts = mt19937_actions(3, 8, 300)
    for t in range(300):
        ref.act(acts[t])
        dut.act(acts[t])
        assert_same_observation(ref, dut, t + 1)
        followed |= dut.info["level_seed"] == np.arange(8) + 4000 + 997
    assert followed.any()
    ref.close()
    dut.close()


def test_array_requested_but_unused_changes_nothing(ref_lib, hostsim_lib):
    ref, dut = make_pair(hostsim_lib, 16, ALL16, launch_shape=(3, False), **KW)
    seeds = next_level_seeds(dut)
    run_lockstep(ref, dut, 200)
    assert (read_lib_array(seeds) == -1).all()
    ref.close()
    dut.close()


def test_entries_consumed_kept_and_untouched_by_set_state(ref_lib, hostsim_lib):
    check_consumed_kept_and_set_state(hostsim_lib)


def test_blob_patcher_rewrites_only_the_named_fields(ref_lib):
    from oracle.ref_env import RefVecEnv

    env = RefVecEnv(2, "heist", **KW)
    env.act(np.array([1, 2], np.int32))
    blob = env.get_state(1)
    st = parse(blob)
    new = patch_fields(blob, reward=2.5, done=1, current_level_seed=77, episodes_remaining=1, prev_level_seed=9, cur_time=3)
    assert len(new) == len(blob)
    got = parse(new)
    want = dict(st, reward=2.5, done=1, current_level_seed=77, episodes_remaining=1, prev_level_seed=9, cur_time=3)
    assert got == want
    offs = field_offsets(blob)
    assert all(parse(patch_fields(blob, **{k: 0}))[k] == 0 for k in offs)
    env.close()
