"""Level generation swept over the seed range: seed lists and the lockstep driver.

Every level an env plays is generated from its level seed alone, so a sweep needs no long runs: the
per-env override (pgb200_get_next_level_seeds) puts every env of a handle on a chosen seed in one step with
action -1, and the reference plays the same step through emulate_step (level_seed_oracle.py). Each batch
of seeds is then compared byte for byte (state blobs: grid, entities, both RNGs, per-game tail) right after
generation and again after a short rollout, outputs at every step."""
import ctypes as C
import json
import os
import zlib

import numpy as np

from helpers import assert_same_observation, read_lib_array, write_lib_array
from level_seed_oracle import emulate_step, next_level_seeds
from oracle.ref_env import mt19937_actions

HERE = os.path.dirname(os.path.abspath(__file__))
# the oracle's records of tests/test_gpu_level_sweep.py, in a file of their own (oracle.record.use_records)
LEVEL_SWEEP_RECORDS = os.path.join(HERE, "golden", "level_sweep_records.json.gz")
# the seeds of the fullest levels of every (game, mode) pair, written by tests/tools/level_extremes.py
LEVEL_EXTREMES = os.path.join(HERE, "golden", "level_extremes.json")

GAMES = ["bigfish", "bossfight", "caveflyer", "chaser", "climber", "coinrun", "dodgeball", "fruitbot", "heist", "jumper",
         "leaper", "maze", "miner", "ninja", "plunder", "starpilot"]
ALL16 = ",".join(GAMES)
# every (game, distribution mode) pair the reference accepts (game.cpp:56-66)
PAIRS = ([(g, "easy") for g in GAMES] + [(g, "hard") for g in GAMES]
         + [(g, "extreme") for g in ("chaser", "dodgeball", "leaper", "starpilot")]
         + [(g, "memory") for g in ("caveflyer", "dodgeball", "heist", "jumper", "maze", "miner")])
# the games with a whole-world view (center_agent=False) and the modes each accepts
WHOLE_WORLD = [("coinrun", "easy"), ("coinrun", "hard"), ("climber", "easy"), ("climber", "hard"), ("caveflyer", "easy"),
               ("caveflyer", "hard"), ("caveflyer", "memory"), ("ninja", "easy"), ("ninja", "hard"), ("jumper", "easy"),
               ("jumper", "hard"), ("jumper", "memory")]

# seeds where an off-by-one in a seed's bits or in the sequential +997 would show
EDGE_SEEDS = ([0, 1, 2, 996, 997, 998] + [v for k in range(8, 31) for v in (2 ** k - 1, 2 ** k)]
              + [2 ** 31 - 998, 2 ** 31 - 2, 2 ** 31 - 1])


def extreme_seeds(game, mode):
    """The seeds of the fullest levels of (game, mode) that tests/tools/level_extremes.py found."""
    with open(LEVEL_EXTREMES) as f:
        pairs = json.load(f)["pairs"]
    out = []
    for g in game.split(","):
        for top in pairs.get(f"{g}/{mode}", {}).values():
            out += [s for _, s in top]
    return out


def sweep_seeds(game, mode, count):
    """`count` level seeds for (game, mode), always the same: the edge seeds, the seeds of the fullest levels,
    then uniform draws over [0, 2^31) from a RandomState keyed by (game, mode)."""
    seeds = list(dict.fromkeys(EDGE_SEEDS + extreme_seeds(game, mode)))
    rs = np.random.RandomState(zlib.crc32(f"{game}/{mode}".encode()))
    seen = set(seeds)
    while len(seeds) < count:
        s = int(rs.randint(0, 2 ** 31))
        if s not in seen:
            seen.add(s)
            seeds.append(s)
    return seeds[:count]


def device_errors(dut):
    dut.lib.pgb200_get_errors.restype = C.c_uint32
    return dut.lib.pgb200_get_errors(C.c_void_p(dut.h), None)


def assert_same_blobs(ref, dut, label):
    for e in range(dut.num):
        assert dut.get_state(e) == ref.get_state(e), f"{label} env {e}: state blobs differ"


def run_level_sweep(ref, dut, seeds, rollout, action_seed=0):
    """ref (the oracle, or its records) and dut (the library under test), both libenv-ABI envs of dut.num envs,
    in batches of dut.num seeds (the last one padded by repeating seeds). For each batch: every env is put
    on its seed (override + action -1; emulate_step on ref), outputs are compared, info level_seed must be
    the seeds and the override array must read -1 again; every env's state blob must be byte-identical;
    then `rollout` lockstep steps of mt19937 actions (outputs every step, blobs at the end). The device's
    error bits must stay 0. Returns the number of batches."""
    n = dut.num
    arr = next_level_seeds(dut)
    assert (read_lib_array(arr) == -1).all(), "a new override array holds -1 everywhere"
    force = np.full(n, -1, np.int32)
    assert_same_observation(ref, dut, "initial reset")
    batches = 0
    for b in range(0, len(seeds), n):
        batch = np.resize(np.asarray(seeds[b:b + n], np.int64), n)
        label = f"seeds {b}..{b + n - 1} ({batch[0]}, ...)"
        write_lib_array(arr, batch)
        _, took = emulate_step(ref, force, batch)
        assert took == list(range(n)), f"{label}: the reference did not reset every env"
        dut.act(force)
        assert_same_observation(ref, dut, label)
        assert np.array_equal(dut.info["level_seed"], batch), f"{label}: info level_seed is not the chosen seeds"
        assert (read_lib_array(arr) == -1).all(), f"{label}: the override array was not consumed"
        assert_same_blobs(ref, dut, f"{label}, generated:")
        acts = mt19937_actions(action_seed + batches, n, rollout)
        for t in range(rollout):
            ref.act(acts[t])
            dut.act(acts[t])
            assert_same_observation(ref, dut, f"{label}, step {t}")
        assert_same_blobs(ref, dut, f"{label}, after {rollout} steps:")
        err = device_errors(dut)
        assert err == 0, f"{label}: device latched error bits {err:#x} (capacity overflow / unsupported feature)"
        batches += 1
    return batches


def sequential_wrap_seeds(n):
    """Overrides 2^31 - 1 - 997 j, j = env % 4: with use_sequential_levels, the level seed passes 2^31 - 1 and
    wraps to a negative seed (game.cpp:99) after j + 1 levels completed in a row."""
    return [2 ** 31 - 1 - 997 * (e % 4) for e in range(n)]


def run_sequential_wrap(ref, dut, steps, action_seed=0):
    """Every env put on sequential_wrap_seeds, then `steps` lockstep steps of mt19937 actions, outputs every
    step and blobs every 50 steps and at the end. Returns the envs that reached a negative level seed."""
    n = dut.num
    arr = next_level_seeds(dut)
    seeds = np.array(sequential_wrap_seeds(n), np.int64)
    force = np.full(n, -1, np.int32)
    assert_same_observation(ref, dut, "initial reset")
    write_lib_array(arr, seeds)
    emulate_step(ref, force, seeds)
    dut.act(force)
    assert_same_observation(ref, dut, "overrides")
    assert np.array_equal(dut.info["level_seed"], seeds)
    wrapped = np.zeros(n, bool)
    acts = mt19937_actions(action_seed, n, steps)
    for t in range(steps):
        ref.act(acts[t])
        dut.act(acts[t])
        assert_same_observation(ref, dut, t)
        wrapped |= dut.info["level_seed"] < 0
        if t % 50 == 49:
            assert_same_blobs(ref, dut, f"step {t}:")
    assert_same_blobs(ref, dut, "end:")
    assert device_errors(dut) == 0
    return np.nonzero(wrapped)[0]
