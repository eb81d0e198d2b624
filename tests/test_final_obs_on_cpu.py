"""Final outputs (pgb200_get_final_outputs) in the host debug build, against the live oracle: every step the outputs,
level_end of every env and the final frames of the envs whose level ended equal the oracle's (its final frames come
from the final-frame hook on a scratch handle, final_obs_oracle.py), and state blobs are compared every 25 steps."""
import numpy as np
import pytest

from final_obs_oracle import force_plan, near_timeout, oracle_final, run_final_lockstep
from helpers import make_pair
from level_seed_oracle import refill_plan
from oracle.ref_env import default_pack

ALL16 = "bigfish,bossfight,caveflyer,chaser,climber,coinrun,dodgeball,fruitbot,heist,jumper,leaper,maze,miner,ninja,plunder,starpilot"
KW = dict(distribution_mode="hard", num_levels=200, start_level=0, rand_seed=0)


def _pair(lib, n, name, launch_shape=None, **kw):
    ref, dut = make_pair(lib, n, name, launch_shape=launch_shape, **kw)
    return ref, oracle_final(ref, n, name, default_pack(), **kw), dut


def _close(*envs):
    for e in envs:
        e.close()


def test_sixteen_games_game_and_caller_ends(ref_lib, hostsim_lib):
    """Every game in hard mode, one action in 16 set to -1: levels ended by the game and by the caller."""
    ref, fin, dut = _pair(hostsim_lib, 16, ALL16, **KW)
    ends = run_final_lockstep(ref, fin, dut, 300, plan=force_plan(1))
    assert (ends == 1).any() and (ends == 3).any()
    _close(ref, fin, dut)


def test_timeout_in_every_game(ref_lib, hostsim_lib):
    """cur_time patched to 10 steps before the time limit in every env of the 16-game list: every game reaches it."""
    n = 32
    ref, fin, dut = _pair(hostsim_lib, n, ALL16, **KW)
    near_timeout([ref, dut], n)
    ends = run_final_lockstep(ref, fin, dut, 40)
    timed_out = {e % 16 for e in np.nonzero((ends == 2).any(0))[0]}
    assert timed_out == set(range(16)), f"games without a timeout: {sorted(set(range(16)) - timed_out)}"
    _close(ref, fin, dut)


def test_sequential_levels(ref_lib, hostsim_lib):
    """use_sequential_levels: a completed maze level goes on with first = 0 and reports level_end = 1."""
    kw = dict(distribution_mode="easy", num_levels=3, start_level=0, rand_seed=0, use_sequential_levels=True)
    ref, fin, dut = _pair(hostsim_lib, 8, "maze", **kw)
    ends = run_final_lockstep(ref, fin, dut, 300, sequential=True)
    assert (ends == 1).any()
    _close(ref, fin, dut)


@pytest.mark.parametrize("name", ["coinrun", "climber", "caveflyer", "ninja", "jumper"])
def test_whole_world_view(ref_lib, hostsim_lib, name):
    kw = dict(KW, center_agent=False)
    ref, fin, dut = _pair(hostsim_lib, 8, name, **kw)
    ends = run_final_lockstep(ref, fin, dut, 150, plan=force_plan(2, every=8))
    assert ends.any()
    _close(ref, fin, dut)


def test_overrides_refilled_every_step(ref_lib, hostsim_lib):
    """Level choice at the same time: the final frame is rendered before the reset that takes the override."""
    ref, fin, dut = _pair(hostsim_lib, 32, ALL16, **KW)
    ends = run_final_lockstep(ref, fin, dut, 200, plan=refill_plan(32, 1), overrides=True)
    assert (ends == 3).any()
    _close(ref, fin, dut)


@pytest.mark.parametrize("chunks", [3, 64])
def test_forced_launch_shapes(ref_lib, hostsim_lib, chunks):
    """Uneven chunks (3 per game) and empty ones (64 per game over 2 envs per game): each launch's own list."""
    n = 48 if chunks == 3 else 32
    ref, fin, dut = _pair(hostsim_lib, n, ALL16, launch_shape=(chunks, False), **KW)
    ends = run_final_lockstep(ref, fin, dut, 150, plan=force_plan(3))
    assert ends.any()
    _close(ref, fin, dut)


def test_game_end_at_the_time_limit(ref_lib, hostsim_lib):
    """Every 4th step every env of the 16-game list starts one step before its time limit, so the levels the game
    ends in those steps end at the limit too: the game's own end takes precedence (game.cpp:134), level_end = 1."""
    n = 64
    ref, fin, dut = _pair(hostsim_lib, n, ALL16, **KW)

    def before(t):
        if t % 4 == 0:
            near_timeout([ref, dut], n, steps_left=1)

    ends = run_final_lockstep(ref, fin, dut, 200, before=before, blob_every=4)
    at_limit = ends[::4]
    assert (at_limit != 0).all() and (at_limit == 1).sum() > 0 and (at_limit == 2).sum() > 0
    _close(ref, fin, dut)
