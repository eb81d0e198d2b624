"""The level bank (pgb200_build_level_bank) in the host debug build.

Reset independence (the field audit): a banked handle and an unbanked one of the same configuration are stepped in
lockstep from many different prior states (random rollouts of different lengths, deaths, time limits spread over the
run, action -1), with num_levels = 200 and a bank over [0, 200), so that every reset is a bank hit. The full state
blob of every env that starts an episode must equal the unbanked one: a header field, an entity, a grid cell, the
RNG or a scratch word that the copy gets wrong shows up here. Then lockstep runs against the live oracle: every game,
the 16-game list, the whole-world view, sequential levels, overrides onto banked and unbanked seeds, final outputs,
the pause mask, forced launch shapes, set_state of a blob made under other options, and in-place rebuilds."""
import numpy as np
import pytest

from final_obs_oracle import force_plan, oracle_final, run_final_lockstep
from helpers import assert_same_observation, make_pair
from level_bank import bank_info, build_bank, error_bits, force_resets, run_bank_lockstep
from level_seed_oracle import patch_fields, refill_plan, run_override_lockstep
from oracle.ref_env import RefVecEnv, default_pack, mt19937_actions
from oracle.state_blob import parse
from pause_oracle import halves_plan, run_pause_lockstep

ALL16 = "bigfish,bossfight,caveflyer,chaser,climber,coinrun,dodgeball,fruitbot,heist,jumper,leaper,maze,miner,ninja,plunder,starpilot"
GAMES = ALL16.split(",")
KW = dict(distribution_mode="hard", num_levels=200, start_level=0, rand_seed=0)
BANK = range(200)


def _close(*envs):
    for e in envs:
        e.close()


def _banked_pair(lib, n, name, seeds=BANK, **kw):
    """(unbanked, banked) handles of the library, same configuration"""
    kw = dict(kw, lib_path=lib, resource_root=default_pack())
    ctrl, banked = RefVecEnv(n, name, **kw), RefVecEnv(n, name, **kw)
    assert build_bank(banked, seeds) == 0
    return ctrl, banked


def _banked_oracle_pair(lib, n, name, seeds=BANK, **kw):
    ref, dut = make_pair(lib, n, name, **kw)
    assert build_bank(dut, seeds) == 0
    return ref, dut


def _spread_time_limits(envs, n, rs):
    """Each env a random 5-120 steps before its time limit (the same states in every handle of `envs`)"""
    for e in range(n):
        blob = envs[0].get_state(e)
        blob = patch_fields(blob, cur_time=max(parse(blob)["timeout"] - int(rs.randint(5, 120)), 0))
        for env in envs:
            env.set_state(e, blob)


@pytest.mark.parametrize("mode", ["easy", "hard"])
@pytest.mark.parametrize("name", GAMES)
def test_reset_independence(hostsim_lib, name, mode):
    n = 16
    ctrl, banked = _banked_pair(hostsim_lib, n, name, **dict(KW, distribution_mode=mode))
    rs = np.random.RandomState(GAMES.index(name))
    # prior states: a rollout of a different length per env before the time limits are spread
    warm = mt19937_actions(1, n, 40)
    for t in range(40):
        a = warm[t].copy()
        a[rs.randint(n)] = -1
        ctrl.act(a)
        banked.act(a)
    _spread_time_limits([ctrl, banked], n, rs)
    starts = run_bank_lockstep(ctrl, banked, 160, plan=force_resets(2, 12), blob_every=40)
    assert starts >= n, f"only {starts} episode starts"
    _close(ctrl, banked)


def test_every_game_against_the_oracle(ref_lib, hostsim_lib):
    for name in GAMES:
        ref, dut = _banked_oracle_pair(hostsim_lib, 8, name, **KW)
        run_bank_lockstep(ref, dut, 100, plan=force_resets(3, 10), blob_every=25, check_errors=False)
        assert not error_bits(dut).any()
        _close(ref, dut)


def test_sixteen_game_list(ref_lib, hostsim_lib):
    ref, dut = _banked_oracle_pair(hostsim_lib, 32, ALL16, **dict(KW, distribution_mode="easy"))
    run_bank_lockstep(ref, dut, 150, plan=force_resets(4, 10), check_errors=False)
    assert not error_bits(dut).any()
    _close(ref, dut)


@pytest.mark.parametrize("name", ["coinrun", "climber", "caveflyer", "ninja", "jumper"])
def test_whole_world_view(ref_lib, hostsim_lib, name):
    ref, dut = _banked_oracle_pair(hostsim_lib, 8, name, **dict(KW, center_agent=False))
    run_bank_lockstep(ref, dut, 80, plan=force_resets(5, 10), check_errors=False)
    _close(ref, dut)


def test_sequential_levels_leave_the_bank(ref_lib, hostsim_lib):
    """Completed levels chain on by +997, out of [0, 200): those resets generate, the rest copy."""
    kw = dict(KW, distribution_mode="easy", use_sequential_levels=True)
    ref, dut = _banked_oracle_pair(hostsim_lib, 8, "maze", **kw)
    run_bank_lockstep(ref, dut, 250, plan=force_resets(6, 40), blob_every=10, check_errors=False)
    _close(ref, dut)


def test_overrides_onto_banked_and_unbanked_seeds(ref_lib, hostsim_lib):
    ref, dut = _banked_oracle_pair(hostsim_lib, 32, ALL16, **KW)
    assert run_override_lockstep(ref, dut, 80, refill_plan(32, 1, low=0, high=400, force_every=4)) > 100
    _close(ref, dut)


def test_final_outputs(ref_lib, hostsim_lib):
    n = 32
    ref, dut = _banked_oracle_pair(hostsim_lib, n, ALL16, **KW)
    fin = oracle_final(ref, n, ALL16, default_pack(), **KW)
    ends = run_final_lockstep(ref, fin, dut, 80, plan=force_plan(7, every=8), blob_every=10)
    assert (ends != 0).sum() > n
    _close(ref, fin, dut)


def test_pause_mask(ref_lib, hostsim_lib):
    n = 32
    ref, dut = _banked_oracle_pair(hostsim_lib, n, ALL16, **KW)
    run_pause_lockstep(ref, dut, 80, halves_plan(n, 8), plan=force_plan(8, every=6), blob_every=5)
    _close(ref, dut)


@pytest.mark.parametrize("chunks", [3, 64])
def test_forced_launch_shapes(ref_lib, hostsim_lib, chunks):
    n = 48 if chunks == 3 else 32
    ref, dut = make_pair(hostsim_lib, n, ALL16, launch_shape=(chunks, False), **KW)
    assert build_bank(dut, BANK) == 0
    run_bank_lockstep(ref, dut, 60, plan=force_resets(9, 8), check_errors=False)
    _close(ref, dut)


def test_set_state_under_other_options_generates(hostsim_lib):
    """A blob made under another distribution_mode carries its options: the env's next resets must generate under
    them, so the bank (made with the handle's options) must not be used for it. The control is an unbanked handle
    (the reference itself cannot play every such blob: it asserts on a grid of the other mode's size)."""
    n = 8
    for name in ("coinrun", "maze", "dodgeball", "chaser", "bossfight", "miner"):
        ctrl, banked = _banked_pair(hostsim_lib, n, name, **dict(KW, distribution_mode="easy"))
        donor = RefVecEnv(n, name, **dict(KW, distribution_mode="hard", rand_seed=3, lib_path=hostsim_lib, resource_root=default_pack()))
        for e in range(0, n, 2):
            blob = donor.get_state(e)
            ctrl.set_state(e, blob)
            banked.set_state(e, blob)
        assert_same_observation(ctrl, banked, "after set_state")
        run_bank_lockstep(ctrl, banked, 60, plan=force_resets(10, 5), blob_every=5)
        _close(ctrl, banked, donor)


def test_rebuild_in_place_between_steps(ref_lib, hostsim_lib):
    n = 32
    ref, dut = _banked_oracle_pair(hostsim_lib, n, ALL16, seeds=range(0, 100), **KW)
    assert bank_info(dut)[0] == 100
    run_bank_lockstep(ref, dut, 30, plan=force_resets(11, 5), check_errors=False)
    assert build_bank(dut, range(100, 200)) == 0
    assert bank_info(dut)[0] == 100
    run_bank_lockstep(ref, dut, 30, plan=force_resets(12, 5), action_seed=1, check_errors=False)
    assert build_bank(dut, []) == 0
    assert bank_info(dut)[0] == 0
    run_bank_lockstep(ref, dut, 20, plan=force_resets(13, 5), action_seed=2, check_errors=False)
    assert not error_bits(dut).any()
    _close(ref, dut)
