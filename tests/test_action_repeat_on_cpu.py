"""Action repeat (pgb200_get_action_repeat) in the host debug build, against the live oracle: every step, each env's
game steps are played on the oracle one plain step at a time, with the envs that are not to play one set back to
their state before it (action_repeat_oracle.py). Outputs and state blobs are compared every step."""
import numpy as np
import pytest

from action_repeat_oracle import action_repeat, constant_plan, mixed_plan, run_repeat_lockstep
from final_obs_oracle import force_plan, near_timeout, oracle_final
from helpers import make_pair, read_lib_array
from level_bank import build_bank
from level_lookahead import enable_lookahead
from level_seed_oracle import refill_plan
from oracle.ref_env import RefVecEnv, default_pack, mt19937_actions
from pause_oracle import halves_plan
from rollout import RolloutCheck

ALL16 = "bigfish,bossfight,caveflyer,chaser,climber,coinrun,dodgeball,fruitbot,heist,jumper,leaper,maze,miner,ninja,plunder,starpilot"
GAMES = ALL16.split(",")
KW = dict(distribution_mode="hard", num_levels=200, start_level=0, rand_seed=0)


def _close(*envs):
    for e in envs:
        e.close()


@pytest.mark.parametrize("mode", ["easy", "hard"])
@pytest.mark.parametrize("name", GAMES)
def test_every_game_mixed_counts(ref_lib, hostsim_lib, name, mode):
    ref, dut = make_pair(hostsim_lib, 8, name, **dict(KW, distribution_mode=mode))
    hist = run_repeat_lockstep(ref, dut, 30, mixed_plan(8, 1))
    assert (hist > 1).any() and (hist == 1).any()
    _close(ref, dut)


def test_sixteen_game_list(ref_lib, hostsim_lib):
    ref, dut = make_pair(hostsim_lib, 32, ALL16, **KW)
    run_repeat_lockstep(ref, dut, 40, mixed_plan(32, 2))
    _close(ref, dut)


@pytest.mark.parametrize("name", ["coinrun", "climber", "caveflyer", "ninja", "jumper"])
def test_whole_world_view(ref_lib, hostsim_lib, name):
    ref, dut = make_pair(hostsim_lib, 8, name, **dict(KW, center_agent=False))
    run_repeat_lockstep(ref, dut, 25, mixed_plan(8, 3))
    _close(ref, dut)


def test_sequential_levels(ref_lib, hostsim_lib):
    """A completed level goes on with first = 0; it still ends the env's game steps of the step."""
    kw = dict(distribution_mode="easy", num_levels=3, start_level=0, rand_seed=0, use_sequential_levels=True)
    ref, dut = make_pair(hostsim_lib, 8, "maze", **kw)
    run_repeat_lockstep(ref, dut, 80, mixed_plan(8, 4, choices=(1, 4, 8, 16)))
    _close(ref, dut)


def test_counts_above_the_time_limit(ref_lib, hostsim_lib):
    """Ten game steps before every env's limit, counts far above it: every env stops at its level's end, within ten
    game steps, whatever its count."""
    n = 16
    ref, dut = make_pair(hostsim_lib, n, ALL16, **KW)
    near_timeout([ref, dut], n)
    huge = np.array([5000, 2 ** 31 - 1, 1001, 10 ** 6] * (n // 4), np.int32)
    hist = run_repeat_lockstep(ref, dut, 6, lambda t: huge if t == 0 else mixed_plan(n, 5)(t))
    assert hist[0].max() <= 10 and (hist[0] > 1).any()
    _close(ref, dut)


def test_action_minus_one(ref_lib, hostsim_lib):
    """Action -1 ends the level in the first game step, whatever the count"""
    n = 16
    ref, dut = make_pair(hostsim_lib, n, ALL16, **KW)
    forced = force_plan(6, every=4)
    hist = run_repeat_lockstep(ref, dut, 30, constant_plan(n, 5), plan=forced)
    assert (hist == 1).any() and (hist > 1).any()
    _close(ref, dut)


def test_overrides_refilled_every_step(ref_lib, hostsim_lib):
    """Level choice at the same time: the one reset of a step takes the env's override"""
    ref, dut = make_pair(hostsim_lib, 32, ALL16, **KW)
    run_repeat_lockstep(ref, dut, 40, mixed_plan(32, 7), plan=refill_plan(32, 1, force_every=6), overrides=True)
    _close(ref, dut)


def test_final_outputs(ref_lib, hostsim_lib):
    """The final frame is the state the level ended in, after the game steps before it; level_end is the last game
    step's"""
    n = 16
    ref, dut = make_pair(hostsim_lib, n, ALL16, **KW)
    fin = oracle_final(ref, n, ALL16, default_pack(), **KW)
    near_timeout([ref, dut], n, steps_left=20)
    run_repeat_lockstep(ref, dut, 30, mixed_plan(n, 8), plan=force_plan(9, every=12), final=fin)
    _close(ref, fin, dut)


def test_pause_mask(ref_lib, hostsim_lib):
    """A paused env plays no game step, whatever its count"""
    n = 32
    ref, dut = make_pair(hostsim_lib, n, ALL16, **KW)
    run_repeat_lockstep(ref, dut, 40, mixed_plan(n, 10), pause_plan=halves_plan(n, 11), plan=force_plan(12, every=10))
    _close(ref, dut)


def test_pause_mask_with_final_outputs(ref_lib, hostsim_lib):
    n = 16
    ref, dut = make_pair(hostsim_lib, n, ALL16, **KW)
    fin = oracle_final(ref, n, ALL16, default_pack(), **KW)
    near_timeout([ref, dut], n, steps_left=15)
    run_repeat_lockstep(ref, dut, 25, mixed_plan(n, 13), pause_plan=halves_plan(n, 14), final=fin)
    _close(ref, fin, dut)


@pytest.mark.parametrize("chunks", [3, 64])
def test_forced_launch_shapes(ref_lib, hostsim_lib, chunks):
    n = 48 if chunks == 3 else 32
    ref, dut = make_pair(hostsim_lib, n, ALL16, launch_shape=(chunks, False), **KW)
    run_repeat_lockstep(ref, dut, 25, mixed_plan(n, 15))
    _close(ref, dut)


def test_level_bank(ref_lib, hostsim_lib):
    """A banked handle's resets run in phase B: the reward after the reset joins the sum there"""
    n = 16
    ref, dut = make_pair(hostsim_lib, n, ALL16, **dict(KW, num_levels=4))
    assert build_bank(dut, list(range(4))) == 0
    near_timeout([ref, dut], n, steps_left=15)
    run_repeat_lockstep(ref, dut, 30, mixed_plan(n, 16), plan=force_plan(17, every=10))
    _close(ref, dut)


def test_level_lookahead(ref_lib, hostsim_lib):
    n = 16
    ref, dut = make_pair(hostsim_lib, n, ALL16, **KW)
    assert enable_lookahead(dut) == 0
    near_timeout([ref, dut], n, steps_left=15)
    run_repeat_lockstep(ref, dut, 30, mixed_plan(n, 18), plan=force_plan(19, every=10))
    _close(ref, dut)


def test_rollout(ref_lib, hostsim_lib):
    """The rollout moves on once per step and holds the step's outputs: the summed rew, the last frame and first"""
    n = 16
    ref, dut = make_pair(hostsim_lib, n, ALL16, **KW)
    fin = oracle_final(ref, n, ALL16, default_pack(), **KW)
    near_timeout([ref, dut], n, steps_left=15)
    roll = RolloutCheck(dut, 3)

    def after_each(t):
        if t > 0:
            rew, ob, first = dut.observe()
            roll.check(t - 1, rew, ob["rgb"], first)

    run_repeat_lockstep(ref, dut, 20, mixed_plan(n, 20), plan=force_plan(21, every=10), final=fin, before=after_each)
    rew, ob, first = dut.observe()
    roll.check(19, rew, ob["rgb"], first)
    _close(ref, fin, dut)


def test_set_state_between_steps(ref_lib, hostsim_lib):
    """set_state of another handle's states between repeated steps: the counts stay, and the loaded envs go on from
    the loaded state"""
    n = 8
    ref, dut = make_pair(hostsim_lib, n, "coinrun", **KW)
    donor = RefVecEnv(n, "coinrun", **dict(KW, rand_seed=7))
    for a in mt19937_actions(3, n, 20):
        donor.act(a)
    blobs = [donor.get_state(e) for e in range(n)]

    def before(t):
        if t == 10:
            for e in range(0, n, 2):
                ref.set_state(e, blobs[e])
                dut.set_state(e, blobs[e])

    run_repeat_lockstep(ref, dut, 25, mixed_plan(n, 22), before=before)
    _close(ref, dut, donor)


def test_all_ones_equals_no_repeat(hostsim_lib):
    """A handle whose counts are all 1 gives, byte for byte, the outputs and states of one that never asked"""
    kw = dict(KW, num_levels=0, resource_root=default_pack(), lib_path=hostsim_lib)
    plain = RefVecEnv(32, ALL16, **kw)
    ones = RefVecEnv(32, ALL16, **kw)
    rep = action_repeat(ones)
    assert rep.dtype == np.int32 and rep.shape == (32,) and (rep == 1).all()
    acts = mt19937_actions(1, 32, 100)
    acts[np.random.RandomState(2).randint(16, size=acts.shape) == 0] = -1
    for t in range(100):
        plain.act(acts[t])
        ones.act(acts[t])
        r1, o1, f1 = plain.observe()
        r2, o2, f2 = ones.observe()
        assert r1.tobytes() == r2.tobytes() and f1.tobytes() == f2.tobytes(), f"step {t}"
        assert o1["rgb"].tobytes() == o2["rgb"].tobytes(), f"step {t}: rgb"
        for k in plain.info:
            assert plain.info[k].tobytes() == ones.info[k].tobytes(), f"step {t}: info {k}"
        if t % 10 == 0:
            for e in range(32):
                assert plain.get_state(e) == ones.get_state(e), f"step {t} env {e}"
    assert (read_lib_array(rep) == 1).all()
    _close(plain, ones)
