"""Level lookahead (pgb200_enable_level_lookahead) in the host debug build.

rand_peek_randint against the draws it predicts. Then lockstep runs at num_levels = 0, the unbounded level
distribution lookahead is for: every game in easy and hard against a handle without lookahead, from many different
prior states (random rollouts, action -1, time limits spread over the run), where every reset must be served from a
slot; and against the live oracle: the 16-game list, the whole-world view, sequential levels, overrides, final outputs,
the pause mask, forced launch shapes, lookahead with a bank, and set_state. Every output, every state blob of an env
that resets and every error bit must be the control's, and the counters must account for every reset."""
import os
import subprocess

import numpy as np
import pytest

from final_obs_oracle import force_plan, oracle_final, run_final_lockstep
from helpers import assert_same_observation, lib_array, make_pair, read_lib_array, write_lib_array
from level_bank import build_bank, error_bits, force_resets
from level_lookahead import enable_lookahead, lookahead_info, run_counted_lockstep
from level_seed_oracle import next_level_seeds, patch_fields, refill_plan, run_override_lockstep
from oracle.ref_env import RefVecEnv, default_pack, mt19937_actions
from oracle.state_blob import parse
from pause_oracle import halves_plan, run_pause_lockstep

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ALL16 = "bigfish,bossfight,caveflyer,chaser,climber,coinrun,dodgeball,fruitbot,heist,jumper,leaper,maze,miner,ninja,plunder,starpilot"
GAMES = ALL16.split(",")
KW = dict(distribution_mode="hard", num_levels=0, start_level=0, rand_seed=0)


def _close(*envs):
    for e in envs:
        e.close()


def _pair(lib, n, name, **kw):
    """(without lookahead, with it): handles of the library, same configuration; lookahead turned on later"""
    kw = dict(kw, lib_path=lib, resource_root=default_pack())
    return RefVecEnv(n, name, **kw), RefVecEnv(n, name, **kw)


def _oracle_pair(lib, n, name, **kw):
    ref, dut = make_pair(lib, n, name, **kw)
    assert enable_lookahead(dut) == 0
    return ref, dut


def _spread_time_limits(envs, n, rs):
    """Each env a random 5-120 steps before its time limit (the same states in every handle of `envs`)"""
    for e in range(n):
        blob = envs[0].get_state(e)
        blob = patch_fields(blob, cur_time=max(parse(blob)["timeout"] - int(rs.randint(5, 120)), 0))
        for env in envs:
            env.set_state(e, blob)


def test_rng_peek_known_answers(tmp_path):
    """rand_peek_randint is the next rand_randint for 10^5 draws per seed and range (straight after mt_seed, and
    through positions 623 and 624 of every generation), and "unknown" for a half-twisted state's untwisted word."""
    exe = str(tmp_path / "rng_peek_check")
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-ffp-contract=off", "-I", os.path.join(ROOT, "procgen_b200", "csrc"),
                           os.path.join(ROOT, "tests", "native", "rng_peek_check.cpp"), "-o", exe])
    out = subprocess.run([exe], capture_output=True, text=True)
    assert out.returncode == 0 and out.stdout.startswith("OK"), out.stdout[-2000:]
    assert int(out.stdout.split()[1]) > 2_000_000


@pytest.mark.parametrize("mode", ["easy", "hard"])
@pytest.mark.parametrize("name", GAMES)
def test_lockstep_against_no_lookahead(hostsim_lib, name, mode):
    n = 16
    ctrl, look = _pair(hostsim_lib, n, name, **dict(KW, distribution_mode=mode))
    rs = np.random.RandomState(GAMES.index(name))
    warm = mt19937_actions(1, n, 40)
    for t in range(40):
        a = warm[t].copy()
        a[rs.randint(n)] = -1
        ctrl.act(a)
        look.act(a)
    _spread_time_limits([ctrl, look], n, rs)
    assert enable_lookahead(look) == 0
    assert lookahead_info(look)["bytes"] > 0
    count = run_counted_lockstep(ctrl, look, 160, plan=force_resets(2, 12), blob_every=40)
    assert count >= n, f"only {count} resets"
    info = lookahead_info(look)
    assert info["generated"] == 0 and info["bank"] == 0 and info["served"] == count, info
    _close(ctrl, look)


def test_sixteen_game_list(ref_lib, hostsim_lib):
    ref, dut = _oracle_pair(hostsim_lib, 32, ALL16, **dict(KW, distribution_mode="easy"))
    count = run_counted_lockstep(ref, dut, 150, plan=force_resets(4, 10), check_errors=False)
    assert not error_bits(dut).any()
    assert lookahead_info(dut)["served"] == count > 32


@pytest.mark.parametrize("name", ["coinrun", "climber", "caveflyer", "ninja", "jumper"])
def test_whole_world_view(ref_lib, hostsim_lib, name):
    ref, dut = _oracle_pair(hostsim_lib, 8, name, **dict(KW, center_agent=False))
    count = run_counted_lockstep(ref, dut, 80, plan=force_resets(5, 10), check_errors=False)
    assert lookahead_info(dut)["served"] == count
    _close(ref, dut)


def test_sequential_levels_miss_after_a_completed_level(ref_lib, hostsim_lib):
    """The draw is predicted: a completed level's +997 generates, every other reset is served."""
    ref, dut = _oracle_pair(hostsim_lib, 8, "maze", **dict(KW, distribution_mode="easy", use_sequential_levels=True))
    acts = mt19937_actions(0, 8, 250)
    completed = 0
    assert_same_observation(ref, dut, -1)
    plan = force_resets(6, 40)
    for t in range(250):
        a = acts[t].copy()
        plan(t, a)
        ref.act(a)
        dut.act(a)
        assert_same_observation(ref, dut, t)
        completed += int((ref.info["prev_level_complete"].astype(bool) & ~ref.first.astype(bool)).sum())
    for e in range(8):
        assert ref.get_state(e) == dut.get_state(e)
    info = lookahead_info(dut)
    assert completed > 0 and info["generated"] == completed, (completed, info)
    assert info["served"] > 0
    _close(ref, dut)


def test_overrides_against_the_oracle(ref_lib, hostsim_lib):
    ref, dut = _oracle_pair(hostsim_lib, 32, ALL16, **KW)
    assert run_override_lockstep(ref, dut, 80, refill_plan(32, 1, force_every=4)) > 100
    _close(ref, dut)


def test_override_generates_and_the_next_reset_hits(hostsim_lib):
    """An override does not advance level_seed_rand_gen: the reset that takes it generates, and the slot still holds
    the level of the next draw, which the reset after it plays."""
    n = 1
    ctrl, look = _pair(hostsim_lib, n, "leaper", **KW)
    assert enable_lookahead(look) == 0
    seeds = [next_level_seeds(env) for env in (ctrl, look)]
    for arr in seeds:
        write_lib_array(arr, np.array([12345], np.int32))
    a = np.full(n, -1, np.int32)
    for env in (ctrl, look):
        env.act(a)
    assert_same_observation(ctrl, look, 0)
    assert look.info["level_seed"][0] == 12345
    assert lookahead_info(look)["generated"] == 1
    for env in (ctrl, look):
        env.act(a)
    assert_same_observation(ctrl, look, 1)
    info = lookahead_info(look)
    assert info["generated"] == 1 and info["served"] == 1, info
    assert ctrl.get_state(0) == look.get_state(0)
    _close(ctrl, look)


def test_final_outputs(ref_lib, hostsim_lib):
    n = 32
    ref, dut = _oracle_pair(hostsim_lib, n, ALL16, **KW)
    fin = oracle_final(ref, n, ALL16, default_pack(), **KW)
    ends = run_final_lockstep(ref, fin, dut, 80, plan=force_plan(7, every=8), blob_every=10)
    assert (ends != 0).sum() > n
    info = lookahead_info(dut)
    assert info["generated"] == 0 and info["served"] == (ends != 0).sum(), info
    _close(ref, fin, dut)


def test_pause_mask(ref_lib, hostsim_lib):
    n = 32
    ref, dut = _oracle_pair(hostsim_lib, n, ALL16, **KW)
    run_pause_lockstep(ref, dut, 80, halves_plan(n, 8), plan=force_plan(8, every=6), blob_every=5)
    info = lookahead_info(dut)
    assert info["generated"] == 0 and info["served"] > n, info
    _close(ref, dut)


@pytest.mark.parametrize("chunks", [3, 64])
def test_forced_launch_shapes(ref_lib, hostsim_lib, chunks):
    n = 48 if chunks == 3 else 32
    ref, dut = make_pair(hostsim_lib, n, ALL16, launch_shape=(chunks, False), **KW)
    assert enable_lookahead(dut) == 0
    count = run_counted_lockstep(ref, dut, 60, plan=force_resets(9, 8), check_errors=False)
    assert lookahead_info(dut)["served"] == count
    _close(ref, dut)


def test_with_a_bank(ref_lib, hostsim_lib):
    """Where the bank holds every seed (num_levels = 200, banked whole), every reset is served by the bank and counted
    so; at num_levels = 0, resets onto banked overrides are too, and none generates. Both orders of the two calls."""
    n = 32
    for bank_first in (True, False):
        kw = dict(KW, num_levels=200)
        ref, dut = make_pair(hostsim_lib, n, ALL16, **kw)
        if bank_first:
            assert build_bank(dut, range(200)) == 0
        assert enable_lookahead(dut) == 0
        if not bank_first:
            assert build_bank(dut, range(200)) == 0
        count = run_counted_lockstep(ref, dut, 60, plan=force_resets(3, 6), check_errors=False)
        info = lookahead_info(dut)
        assert info["bank"] == count and info["served"] == 0 and info["generated"] == 0, (count, info)
        _close(ref, dut)
    ref, dut = _oracle_pair(hostsim_lib, n, ALL16, **KW)
    assert build_bank(dut, range(100)) == 0
    taken = run_override_lockstep(ref, dut, 60, refill_plan(n, 2, low=0, high=100, force_every=3))
    info = lookahead_info(dut)
    assert taken > 50 and info["bank"] == taken and info["generated"] == 0, (taken, info)
    _close(ref, dut)


def test_set_state_generates_once(hostsim_lib):
    """An env loaded with another env's blob draws its next seed from the blob's generator: that reset generates,
    and the one after it plays the level generated ahead for it."""
    n = 8
    ctrl, look = _pair(hostsim_lib, n, "caveflyer", **KW)
    donor = RefVecEnv(n, "caveflyer", **dict(KW, rand_seed=7, lib_path=hostsim_lib, resource_root=default_pack()))
    assert enable_lookahead(look) == 0
    for e in range(0, n, 2):
        blob = donor.get_state(e)
        ctrl.set_state(e, blob)
        look.set_state(e, blob)
    a = np.full(n, -1, np.int32)
    for step in range(2):
        for env in (ctrl, look):
            env.act(a)
        assert_same_observation(ctrl, look, step)
        info = lookahead_info(look)
        assert info["generated"] == n // 2 and info["served"] == [n // 2, n // 2 + n][step], info
    for e in range(n):
        assert ctrl.get_state(e) == look.get_state(e)
    _close(ctrl, look, donor)


def test_set_state_under_other_options_generates(hostsim_lib):
    """A blob made under another distribution_mode carries its options: its env's resets generate under them."""
    n = 8
    for name in ("coinrun", "maze", "dodgeball", "chaser", "bossfight", "miner"):
        ctrl, look = _pair(hostsim_lib, n, name, **dict(KW, distribution_mode="easy"))
        donor = RefVecEnv(n, name, **dict(KW, distribution_mode="hard", rand_seed=3, lib_path=hostsim_lib, resource_root=default_pack()))
        assert enable_lookahead(look) == 0
        for e in range(0, n, 2):
            blob = donor.get_state(e)
            ctrl.set_state(e, blob)
            look.set_state(e, blob)
        assert_same_observation(ctrl, look, "after set_state")
        count = run_counted_lockstep(ctrl, look, 60, plan=force_resets(10, 5), blob_every=5)
        info = lookahead_info(look)
        assert info["generated"] > 0 and info["served"] > 0 and info["served"] + info["generated"] == count, info
        _close(ctrl, look, donor)
