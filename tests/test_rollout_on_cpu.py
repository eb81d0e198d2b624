"""The rollout (pgb200_get_rollout) in the host debug build, against controls without it.

A handle with the rollout and one without it step together. After every step their outputs, and every few steps their
state blobs, must be equal, and the rollout must hold its invariant: the cursor has moved on by one slot, that slot holds
the step's rgb, rew and first byte for byte, and every other slot is unchanged. Runs cover more than one wrap of the ring:
every game in easy and hard, the 16-game list, the whole-world view, sequential levels, overrides, final outputs, the
pause mask, forced launch shapes and set_state, which leaves the rollout alone."""
import numpy as np
import pytest

from final_obs_oracle import LibFinal
from helpers import write_lib_array
from level_bank import force_resets
from level_seed_oracle import next_level_seeds
from oracle.ref_env import RefVecEnv, default_pack, mt19937_actions
from pause_oracle import pause_mask
from rollout import RolloutCheck, run_rollout_lockstep

ALL16 = "bigfish,bossfight,caveflyer,chaser,climber,coinrun,dodgeball,fruitbot,heist,jumper,leaper,maze,miner,ninja,plunder,starpilot"
GAMES = ALL16.split(",")
KW = dict(distribution_mode="hard", num_levels=0, start_level=0, rand_seed=0)
SLOTS = 4
STEPS = 2 * SLOTS + 3  # more than two wraps of the ring


def _pair(lib, n, name, **kw):
    """(control, handle the rollout is requested on): handles of the library, same configuration"""
    kw = dict(KW, **kw)
    kw.update(lib_path=lib, resource_root=default_pack())
    return RefVecEnv(n, name, **kw), RefVecEnv(n, name, **kw)


def _close(*envs):
    for e in envs:
        e.close()


@pytest.mark.parametrize("mode", ["easy", "hard"])
@pytest.mark.parametrize("name", GAMES)
def test_every_game(hostsim_lib, name, mode):
    n = 8
    ctrl, dut = _pair(hostsim_lib, n, name, distribution_mode=mode)
    warm = mt19937_actions(1, n, 6)
    for a in warm:  # the first call copies the outputs of the latest step, not of the initial reset
        ctrl.act(a)
        dut.act(a)
    run_rollout_lockstep(ctrl, dut, STEPS, SLOTS, plan=force_resets(GAMES.index(name), 5))
    _close(ctrl, dut)


def test_sixteen_game_list(hostsim_lib):
    ctrl, dut = _pair(hostsim_lib, 32, ALL16, distribution_mode="easy")
    run_rollout_lockstep(ctrl, dut, 3 * 5 + 1, 5, plan=force_resets(4, 6))
    _close(ctrl, dut)


@pytest.mark.parametrize("name", ["coinrun", "climber", "caveflyer", "ninja", "jumper"])
def test_whole_world_view(hostsim_lib, name):
    ctrl, dut = _pair(hostsim_lib, 8, name, center_agent=False)
    run_rollout_lockstep(ctrl, dut, STEPS, SLOTS, plan=force_resets(5, 5))
    _close(ctrl, dut)


def test_sequential_levels(hostsim_lib):
    ctrl, dut = _pair(hostsim_lib, 8, "maze", distribution_mode="easy", use_sequential_levels=True, num_levels=10)
    run_rollout_lockstep(ctrl, dut, 40, 3, plan=force_resets(6, 12))
    _close(ctrl, dut)


def test_overrides(hostsim_lib):
    n = 32
    ctrl, dut = _pair(hostsim_lib, n, ALL16)
    seeds = [next_level_seeds(env) for env in (ctrl, dut)]
    rs = np.random.RandomState(2)

    def before(t, a):
        ov = np.where(rs.randint(3, size=n) == 0, rs.randint(0, 2 ** 31 - 1, size=n), -1).astype(np.int32)
        a[rs.randint(4, size=n) == 0] = -1
        for arr in seeds:
            write_lib_array(arr, ov)

    run_rollout_lockstep(ctrl, dut, STEPS, SLOTS, before=before)
    _close(ctrl, dut)


def test_final_outputs(hostsim_lib):
    """A slot holds the next level's first frame (the step's rgb), not the final frame of the level that ended."""
    n = 32
    ctrl, dut = _pair(hostsim_lib, n, ALL16)
    fins = [LibFinal(env) for env in (ctrl, dut)]
    seen = {"ends": 0}
    state = {}

    def after(t):
        (le_c, rgb_c), (le_d, rgb_d) = (f.read() for f in fins)
        assert np.array_equal(le_c, le_d) and np.array_equal(rgb_c, rgb_d), f"step {t}: final outputs differ"
        ended = le_d != 0
        c = int(state["roll"].prev["cursor"][0])
        slot = state["roll"].prev["rgb"][c]
        assert np.array_equal(slot[ended], dut.observe()[1]["rgb"][ended])
        differs = (slot[ended] != rgb_d[ended]).reshape(int(ended.sum()), -1).any(1)
        seen["ends"] += int(ended.sum())
        seen["differs"] = seen.get("differs", 0) + int(differs.sum())

    state["roll"] = RolloutCheck(dut, SLOTS)
    run_rollout_lockstep(ctrl, dut, STEPS, SLOTS, plan=force_resets(7, 4), after=after, roll=state["roll"])
    assert seen["ends"] > n and seen["differs"] > n // 2, seen
    _close(ctrl, dut)


@pytest.mark.parametrize("final", [False, True])
def test_pause_mask(hostsim_lib, final):
    """A paused env's slot holds the frame it is paused on, with rew = 0 and first = 0."""
    n = 32
    ctrl, dut = _pair(hostsim_lib, n, ALL16)
    if final:
        for env in (ctrl, dut):
            LibFinal(env)
    masks = [pause_mask(env) for env in (ctrl, dut)]
    state = {"paused": np.zeros(n, bool), "checked": 0}

    def before(t, a):
        state["paused"] = np.random.RandomState([8, t]).randint(2, size=n).astype(bool)
        state["prev_rgb"] = dut.observe()[1]["rgb"].copy()
        for m in masks:
            write_lib_array(m, state["paused"])

    def after(t):
        p = state["paused"]
        c = int(roll.prev["cursor"][0])
        assert not roll.prev["rew"][c][p].any() and not roll.prev["first"][c][p].any()
        assert np.array_equal(roll.prev["rgb"][c][p], state["prev_rgb"][p]), f"step {t}: a paused env's slot is not its frame"
        state["checked"] += int(p.sum())

    roll = RolloutCheck(dut, SLOTS)
    run_rollout_lockstep(ctrl, dut, STEPS, SLOTS, plan=force_resets(9, 4), before=before, after=after, roll=roll)
    assert state["checked"] > n
    _close(ctrl, dut)


@pytest.mark.parametrize("chunks,serialize", [(3, False), (64, False), (3, True)])
def test_forced_launch_shapes(hostsim_lib, chunks, serialize):
    n = 48 if chunks == 3 else 32
    ctrl, dut = _pair(hostsim_lib, n, ALL16, launch_shape=(chunks, serialize))
    run_rollout_lockstep(ctrl, dut, STEPS, SLOTS, plan=force_resets(10, 5))
    _close(ctrl, dut)


def test_set_state_leaves_the_rollout_alone(hostsim_lib):
    n = 16
    ctrl, dut = _pair(hostsim_lib, n, ALL16)
    donor = RefVecEnv(n, ALL16, **dict(KW, rand_seed=7, lib_path=hostsim_lib, resource_root=default_pack()))
    for a in mt19937_actions(3, n, 12):
        donor.act(a)
    roll = run_rollout_lockstep(ctrl, dut, SLOTS + 1, SLOTS)
    blobs = [dut.get_state(e) for e in range(n)]
    for e in range(0, n, 2):
        blob = donor.get_state(e)
        ctrl.set_state(e, blob)
        dut.set_state(e, blob)
    roll.unchanged("after set_state")
    for e in range(n):
        assert dut.get_state(e) == (donor.get_state(e) if e % 2 == 0 else blobs[e])
    run_rollout_lockstep(ctrl, dut, STEPS, SLOTS, roll=roll, action_seed=1)
    _close(ctrl, dut, donor)
