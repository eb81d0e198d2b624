"""get_state / set_state of chosen envs (pgb200_get_states / pgb200_set_states) in the host debug build, against the
live oracle.

For every game and mode (all 16 games easy and hard, the extreme and memory modes where a game has them, the 16-game
list, the whole-world view, sequential levels): the blobs of a random, unsorted list of envs with a duplicate are the
oracle's, byte for byte; blobs of another handle (other seed, other time) loaded into a random subset leave the
library where the oracle's set_state leaves the oracle, and the two then run in lockstep for 50 steps, blobs compared
every step; the envs outside the subset run on as a twin handle that never restored. Then the same restore with every
opt-in of the step on, and set_state's refusals sent in the middle of a batch."""
import os
import subprocess
import sys
import zlib
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

from helpers import assert_same_observation, lib_array, make_pair, read_lib_array
from level_bank import build_bank
from level_lookahead import enable_lookahead, lookahead_info
from level_seed_oracle import next_level_seeds
from oracle.ref_env import RefVecEnv, default_pack, mt19937_actions
from pause_oracle import assert_same_paused_observation, emulate_pause_step, pause_mask
from rollout import RolloutCheck
from state_batch import distinct_subset, get_states, set_states, subset_with_duplicates
from test_state_blob_checks_on_cpu import KW as CHECKS_KW
from test_state_blob_checks_on_cpu import REJECTIONS, state_after_steps

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GAMES = ["bigfish", "bossfight", "caveflyer", "chaser", "climber", "coinrun", "dodgeball", "fruitbot", "heist", "jumper",
         "leaper", "maze", "miner", "ninja", "plunder", "starpilot"]
ALL16 = ",".join(GAMES)
CASES = ([(g, "easy", {}) for g in GAMES] + [(g, "hard", {}) for g in GAMES] +
         [(g, "extreme", {}) for g in ("chaser", "dodgeball", "leaper", "starpilot")] +
         [(g, "memory", {}) for g in ("caveflyer", "dodgeball", "heist", "jumper", "maze", "miner")] +
         [(ALL16, "hard", {})] +
         [(g, "hard", {"center_agent": False}) for g in ("coinrun", "climber", "caveflyer", "jumper", "ninja")] +
         [(g, "hard", {"use_sequential_levels": True}) for g in ("coinrun", "maze", "ninja")])


def _id(case):
    name, mode, extra = case
    return "-".join(["all16" if name == ALL16 else name, mode] + sorted(extra))


def _rest(n, envs):
    return np.setdiff1d(np.arange(n), envs)


@pytest.mark.parametrize("case", CASES, ids=[_id(c) for c in CASES])
def test_states_against_oracle(ref_lib, hostsim_lib, case):
    name, mode, extra = case
    n = 16 if name == ALL16 else 6
    kw = dict(distribution_mode=mode, num_levels=200, start_level=0, rand_seed=0, **extra)
    ref, dut = make_pair(hostsim_lib, n, name, **kw)
    twin = RefVecEnv(n, name, lib_path=hostsim_lib, resource_root=default_pack(), **kw)
    donor = RefVecEnv(n, name, **dict(kw, rand_seed=5))
    rng = np.random.RandomState(zlib.crc32(_id(case).encode()))
    acts = mt19937_actions(0, n, 62)
    for t in range(12):
        for env in (ref, dut, twin):
            env.act(acts[t])
    for a in mt19937_actions(1, n, 17):
        donor.act(a)
    listed = subset_with_duplicates(rng, n, n + 2)
    assert get_states(dut, listed) == [ref.get_state(e) for e in listed]
    # another handle's blobs, each into an env of its game (env e of a list plays game e % 16)
    restored = distinct_subset(rng, n, n // 2)
    blobs = [donor.get_state(e) for e in restored]
    for e, b in zip(restored, blobs):
        ref.set_state(e, b)
    assert set_states(dut, restored, blobs) == 0
    assert_same_observation(ref, dut, "after set_states")
    rest = _rest(n, restored)
    for t in range(12, 62):
        if t > 12:
            for env in (ref, dut, twin):
                env.act(acts[t])
            assert_same_observation(ref, dut, t)
        _, o_dut, _ = dut.observe()
        _, o_twin, _ = twin.observe()
        assert np.array_equal(o_dut["rgb"][rest], o_twin["rgb"][rest]) and np.array_equal(dut.rew[rest], twin.rew[rest])
        assert np.array_equal(dut.first[rest], twin.first[rest])
        got = get_states(dut, list(range(n)))
        assert got == [ref.get_state(e) for e in range(n)], f"step {t}: blobs differ"
        assert [got[e] for e in rest] == get_states(twin, rest), f"step {t}: an env outside the subset changed"
    for env in (ref, dut, twin, donor):
        env.close()


def _final_outputs(env):
    import ctypes as C

    from procgen_b200.libenv import FinalOutputs

    env.lib.pgb200_get_final_outputs.argtypes = [C.c_void_p, C.POINTER(FinalOutputs)]
    env.lib.pgb200_get_final_outputs.restype = C.c_int
    out = FinalOutputs()
    assert env.lib.pgb200_get_final_outputs(C.c_void_p(env.h), C.byref(out)) == 0
    return {"rgb": lib_array(env, out.rgb, (env.num, 64, 64, 3), "|u1"), "level_end": lib_array(env, out.level_end, (env.num,), "|u1")}


def test_restore_with_every_opt_in(ref_lib, hostsim_lib):
    """Final outputs, the rollout, the pause mask, overrides, a bank of half the level set and level lookahead all on.
    set_states into paused and running envs writes nothing of them (the overrides are neither read nor changed) and
    leaves the oracle's outputs; the paused restored envs keep their restored state; then lockstep with the oracle
    through forced resets, in which the restored envs' lookahead slots miss and then serve."""
    n, name = 8, "coinrun"
    kw = dict(distribution_mode="hard", num_levels=50, start_level=0, rand_seed=0)
    ref, dut = make_pair(hostsim_lib, n, name, **kw)
    donor = RefVecEnv(n, name, **dict(kw, rand_seed=5))
    for a in mt19937_actions(1, n, 25):
        donor.act(a)
    final = _final_outputs(dut)
    roll = RolloutCheck(dut, 4)
    mask, seeds = pause_mask(dut), next_level_seeds(dut)
    assert build_bank(dut, range(0, 25)) == 0 and enable_lookahead(dut) == 0
    acts = mt19937_actions(0, n, 80)
    for t in range(10):
        ref.act(acts[t])
        dut.act(acts[t])
        assert_same_observation(ref, dut, t)
        roll.check(t, dut.rew, dut.rgb, dut.first)
    paused = np.zeros(n, bool)
    paused[[1, 2, 5]] = True
    mask[:] = paused
    seeds[:] = 7
    restored = [5, 3, 2, 6]
    blobs = [donor.get_state(e) for e in restored]
    final_before = {k: read_lib_array(v) for k, v in final.items()}
    for e, b in zip(restored, blobs):
        ref.set_state(e, b)
    assert set_states(dut, restored, blobs) == 0
    assert (read_lib_array(seeds) == 7).all() and np.array_equal(read_lib_array(mask), paused)
    roll.unchanged("set_states")
    for k, v in final.items():
        assert np.array_equal(read_lib_array(v), final_before[k]), f"set_states changed the final outputs' {k}"
    assert_same_observation(ref, dut, "after set_states")
    seeds[:] = -1
    for t in range(10, 15):
        emulate_pause_step(ref, acts[t], paused)
        dut.act(acts[t])
        assert_same_paused_observation(ref, dut, paused, t)
        roll.check(t, dut.rew, dut.rgb, dut.first)
        assert get_states(dut, [5, 2]) == [blobs[0], blobs[2]], f"step {t}: a paused restored env moved"
    mask[:] = 0
    before = lookahead_info(dut)
    for t in range(15, 80):
        a = acts[t].copy()
        if t % 8 == 0:
            a[:] = -1
        ref.act(a)
        dut.act(a)
        assert_same_observation(ref, dut, t)
        roll.check(t, dut.rew, dut.rgb, dut.first)
        assert get_states(dut, list(range(n))) == [ref.get_state(e) for e in range(n)], f"step {t}: blobs differ"
    info = lookahead_info(dut)
    assert info["generated"] > before["generated"] and info["served"] > before["served"], (before, info)
    for env in (ref, dut, donor):
        env.close()


SET_STATES = r"""
import sys
sys.path.insert(0, {root!r}); sys.path.insert(0, {root!r} + "/tests")
from oracle.ref_env import RefVecEnv, default_pack
from state_batch import set_states
env = RefVecEnv({n}, {game!r}, lib_path={lib!r}, resource_root=default_pack(), **{kw!r})
good = [env.get_state(e) for e in range(env.num)]
envs = [3, {bad}, 0]
blobs = [open({path!r}, "rb").read() if e == {bad} else good[e] for e in envs]
set_states(env, envs, blobs)
print("set_states returned")
"""


@pytest.fixture(scope="module")
def rejected(hostsim_lib, tmp_path_factory):
    """{case: (exit code, output)} of one set_states of [3, 2, 0] whose middle blob is the case's, each in a process of
    its own. The cases are set_state's (tests/test_state_blob_checks_on_cpu.py), and a coinrun blob sent to env 2 of the
    16-game list, which plays caveflyer."""
    games = sorted({g for g, _, _ in REJECTIONS.values()} | {"coinrun"})
    good = {game: state_after_steps(hostsim_lib, game) for game in games}
    cases = {case: (game, edit(good[game])) for case, (game, edit, _) in REJECTIONS.items()}
    cases["game_list"] = (ALL16, good["coinrun"])
    d = tmp_path_factory.mktemp("batch_blobs")
    for case, (_, blob) in cases.items():
        (d / case).write_bytes(blob)

    def run(case):
        game = cases[case][0]
        script = SET_STATES.format(root=ROOT, n=16 if game == ALL16 else 4, game=game, lib=hostsim_lib, kw=CHECKS_KW,
                                   bad=2, path=str(d / case))
        r = subprocess.run([sys.executable, "-c", script], capture_output=True, text=True, timeout=300)
        return r.returncode, r.stdout + r.stderr

    with ThreadPoolExecutor(max_workers=os.cpu_count() or 4) as ex:
        return dict(zip(cases, ex.map(run, cases)))


@pytest.mark.parametrize("case", list(REJECTIONS) + ["game_list"])
def test_set_states_refuses_a_bad_blob_in_a_batch(rejected, case):
    code, out = rejected[case]
    fatal = [line for line in out.splitlines() if line.startswith("fatal: set_state:")]
    assert code != 0 and fatal, out[-2000:]
    check = "another game" if case == "game_list" else REJECTIONS[case][2]
    assert check in fatal[0] and "(env 2)" in fatal[0], fatal[0]
