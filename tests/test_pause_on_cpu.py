"""The pause mask (pgb200_get_pause_mask) in the host debug build, against the live oracle: every step, a paused env's
step is emulated on the oracle (a plain step, then set_state of its pre-step blob; pause_oracle.py), the outputs are
compared, and every env's state blob before the step is compared."""
import numpy as np
import pytest

from final_obs_oracle import near_timeout, oracle_final
from helpers import make_pair
from level_seed_oracle import refill_plan
from oracle.ref_env import RefVecEnv, default_pack
from pause_oracle import (all_plan, check_set_state_into_paused_env, episode_end_plan, halves_plan, long_plan,
                          run_pause_lockstep, zero_plan)

ALL16 = "bigfish,bossfight,caveflyer,chaser,climber,coinrun,dodgeball,fruitbot,heist,jumper,leaper,maze,miner,ninja,plunder,starpilot"
GAMES = ALL16.split(",")
KW = dict(distribution_mode="hard", num_levels=200, start_level=0, rand_seed=0)


def _close(*envs):
    for e in envs:
        e.close()


@pytest.mark.parametrize("mode", ["easy", "hard"])
@pytest.mark.parametrize("name", GAMES)
def test_every_game_random_halves(ref_lib, hostsim_lib, name, mode):
    ref, dut = make_pair(hostsim_lib, 8, name, **dict(KW, distribution_mode=mode))
    hist = run_pause_lockstep(ref, dut, 60, halves_plan(8, 1))
    assert hist.any() and not hist.all()
    _close(ref, dut)


def test_sixteen_game_list(ref_lib, hostsim_lib):
    """The 16-game list: random halves, then the evaluation pattern with aligned releases."""
    ref, dut = make_pair(hostsim_lib, 32, ALL16, **KW)
    halves, ends = halves_plan(32, 2), episode_end_plan(32, release_every=50)
    run_pause_lockstep(ref, dut, 200, lambda t, first: halves(t, first) if t < 100 else ends(t, first), blob_every=5)
    _close(ref, dut)


def test_long_pauses_span_the_time_limit(ref_lib, hostsim_lib):
    """cur_time 10 steps before the limit, then windows of 20-60 paused steps starting in the first 8: a paused step
    does not count toward the limit, and every env times out 10 running steps after it started."""
    n = 32
    ref, dut = make_pair(hostsim_lib, n, ALL16, **KW)
    near_timeout([ref, dut], n)
    hist = run_pause_lockstep(ref, dut, 80, long_plan(n, 3))
    assert hist.sum(0).min() >= 20
    _close(ref, dut)


def test_pause_at_episode_end(ref_lib, hostsim_lib):
    """The one-episode-per-level evaluation: an env is paused from the step after its level ended, until the end."""
    n = 32
    ref, dut = make_pair(hostsim_lib, n, ALL16, **KW)
    near_timeout([ref, dut], n, steps_left=40)
    hist = run_pause_lockstep(ref, dut, 60, episode_end_plan(n))
    assert hist[-1].all(), "every env's level ended within 41 steps of its limit"
    _close(ref, dut)


def test_every_env_paused(ref_lib, hostsim_lib):
    ref, dut = make_pair(hostsim_lib, 16, ALL16, **KW)
    hist = run_pause_lockstep(ref, dut, 50, all_plan(16))
    assert hist[10:40].all()
    _close(ref, dut)


def test_all_zero_mask_equals_no_mask(ref_lib, hostsim_lib):
    ref, dut = make_pair(hostsim_lib, 16, ALL16, **KW)
    run_pause_lockstep(ref, dut, 100, zero_plan(16), blob_every=10)
    _close(ref, dut)


def test_sequential_levels(ref_lib, hostsim_lib):
    kw = dict(distribution_mode="easy", num_levels=3, start_level=0, rand_seed=0, use_sequential_levels=True)
    ref, dut = make_pair(hostsim_lib, 8, "maze", **kw)
    run_pause_lockstep(ref, dut, 200, halves_plan(8, 4), blob_every=5)
    _close(ref, dut)


@pytest.mark.parametrize("name", ["coinrun", "climber", "caveflyer", "ninja", "jumper"])
def test_whole_world_view(ref_lib, hostsim_lib, name):
    ref, dut = make_pair(hostsim_lib, 8, name, **dict(KW, center_agent=False))
    run_pause_lockstep(ref, dut, 60, halves_plan(8, 5))
    _close(ref, dut)


def test_overrides_refilled_every_step(ref_lib, hostsim_lib):
    """Level choice at the same time: a paused env neither reads nor consumes its override, even with action -1."""
    ref, dut = make_pair(hostsim_lib, 32, ALL16, **KW)
    run_pause_lockstep(ref, dut, 100, halves_plan(32, 6), plan=refill_plan(32, 1, force_every=4), overrides=True, blob_every=5)
    _close(ref, dut)


def test_final_outputs(ref_lib, hostsim_lib):
    """Final outputs at the same time: level_end = 0 on a paused env and its final frame stays; the evaluation
    pattern with forced resets."""
    n = 32
    ref, dut = make_pair(hostsim_lib, n, ALL16, **KW)
    fin = oracle_final(ref, n, ALL16, default_pack(), **KW)
    rs = np.random.RandomState(7)

    def plan(t, actions, pending):
        actions[rs.randint(16, size=n) == 0] = -1
        return {}

    run_pause_lockstep(ref, dut, 100, episode_end_plan(n, release_every=20), plan=plan, final=fin, blob_every=5)
    _close(ref, fin, dut)


@pytest.mark.parametrize("chunks", [3, 64])
def test_forced_launch_shapes(ref_lib, hostsim_lib, chunks):
    n = 48 if chunks == 3 else 32
    ref, dut = make_pair(hostsim_lib, n, ALL16, launch_shape=(chunks, False), **KW)
    run_pause_lockstep(ref, dut, 60, halves_plan(n, 8))
    _close(ref, dut)


def test_action_minus_one_on_paused_envs(ref_lib, hostsim_lib):
    """Every paused env gets action -1, which it ignores."""
    ref, dut = make_pair(hostsim_lib, 16, ALL16, **KW)
    run_pause_lockstep(ref, dut, 60, halves_plan(16, 9), force_paused=True)
    _close(ref, dut)


def test_set_state_into_paused_env(ref_lib, hostsim_lib):
    kw = dict(KW, lib_path=hostsim_lib, resource_root=default_pack())
    dut = RefVecEnv(8, "coinrun", **kw)
    donor = RefVecEnv(8, "coinrun", **dict(kw, rand_seed=7))
    check_set_state_into_paused_env(donor, dut)
    _close(dut, donor)
