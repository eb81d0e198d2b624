"""The level-bank entry points of the C ABI without a GPU: exported by both builds and declared by the header; in the
host debug build, bad seeds and more distinct seeds than the capacity are refused, pgb200_level_bank_info reports the
bank, and an empty bank gives the outputs and states of a handle without one."""
import ctypes as C
import os
import re

import numpy as np

from procgen_b200 import libenv as L

HEADER = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "procgen_b200.h")
ALL16 = "bigfish,bossfight,caveflyer,chaser,climber,coinrun,dodgeball,fruitbot,heist,jumper,leaper,maze,miner,ninja,plunder,starpilot"


def _env(lib, n=16, name=ALL16):
    from oracle.ref_env import RefVecEnv, default_pack

    return RefVecEnv(n, name, distribution_mode="hard", num_levels=200, rand_seed=0, resource_root=default_pack(), lib_path=lib)


def test_exported(product_lib, hostsim_lib):
    for path in (product_lib, hostsim_lib):
        lib = C.CDLL(path)
        assert hasattr(lib, "pgb200_build_level_bank") and hasattr(lib, "pgb200_level_bank_info")
    assert "pgb200_build_level_bank" in L.EXPORTS and "pgb200_level_bank_info" in L.EXPORTS
    text = open(HEADER).read()
    assert re.search(r"LIBENV_API int pgb200_build_level_bank\(libenv_env \*handle, const int32_t \*seeds, int count, int capacity\);", text)
    assert re.search(r"LIBENV_API int pgb200_level_bank_info\(libenv_env \*handle, int \*levels, int64_t \*bytes\);", text)


def test_refusals_and_info(hostsim_lib):
    from level_bank import bank_info, build_bank

    env = _env(hostsim_lib)
    assert bank_info(env) == (0, 0)
    assert build_bank(env, []) == -1, "a first call with no seeds and no capacity"
    assert build_bank(env, [3, -1, 5]) == -1, "a negative seed"
    assert build_bank(env, [2 ** 31 - 1, 0]) == 0  # the edges of [0, 2^31); capacity 2
    assert bank_info(env)[0] == 2
    assert build_bank(env, [1, 2, 3]) == -1, "three distinct seeds, capacity 2"
    assert bank_info(env)[0] == 2, "a refused call changes nothing"
    env.close()

    env = _env(hostsim_lib)
    assert build_bank(env, range(10), capacity=50) == 0
    levels, nbytes = bank_info(env)
    assert levels == 10 and nbytes > 16 * 50 * 4096, "room for 50 levels of every game of the list"
    assert build_bank(env, list(range(50)) * 3) == 0, "duplicates are allowed and count once"
    assert bank_info(env) == (50, nbytes), "a rebuild keeps the capacity and the memory"
    assert build_bank(env, range(51)) == -1
    assert build_bank(env, []) == 0
    assert bank_info(env) == (0, nbytes)
    env.close()


def test_empty_bank_equals_no_bank(hostsim_lib):
    from level_bank import build_bank, force_resets, run_bank_lockstep

    plain, banked = _env(hostsim_lib, 32), _env(hostsim_lib, 32)
    assert build_bank(banked, [], capacity=200) == 0
    run_bank_lockstep(plain, banked, 80, plan=force_resets(1, 6), blob_every=20)
    plain.close()
    banked.close()
