"""The level-lookahead entry points of the C ABI without a GPU: exported by both builds and declared by the header; in
the host debug build, pgb200_level_lookahead_info is all zeros before pgb200_enable_level_lookahead, a second enable
changes nothing, and a closed handle gives back every byte lookahead took from the process's heap."""
import ctypes as C
import os
import re
import subprocess
import sys

import pytest

from procgen_b200 import libenv as L

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "procgen_b200.h")


def _env(lib, n=16, name="coinrun", **kw):
    from oracle.ref_env import RefVecEnv, default_pack

    return RefVecEnv(n, name, **dict(dict(distribution_mode="hard", num_levels=0, rand_seed=0), **kw), resource_root=default_pack(), lib_path=lib)


def test_exported(product_lib, hostsim_lib):
    for path in (product_lib, hostsim_lib):
        lib = C.CDLL(path)
        assert hasattr(lib, "pgb200_enable_level_lookahead") and hasattr(lib, "pgb200_level_lookahead_info")
    assert "pgb200_enable_level_lookahead" in L.EXPORTS and "pgb200_level_lookahead_info" in L.EXPORTS
    text = open(HEADER).read()
    assert re.search(r"LIBENV_API int pgb200_enable_level_lookahead\(libenv_env \*handle\);", text)
    assert re.search(r"LIBENV_API int pgb200_level_lookahead_info\(libenv_env \*handle, int64_t \*out /\* \[4\] \*/\);", text)


def test_info_and_idempotent_enable(hostsim_lib):
    from level_lookahead import enable_lookahead, lookahead_info
    from oracle.ref_env import mt19937_actions

    env = _env(hostsim_lib)
    assert lookahead_info(env) == dict(served=0, bank=0, generated=0, bytes=0)
    assert enable_lookahead(env) == 0
    first = lookahead_info(env)
    assert first["served"] == first["bank"] == first["generated"] == 0
    assert first["bytes"] > 16 * 24 * 1024, "a slot of at least 24 KB per env"
    acts = mt19937_actions(0, 16, 20)
    acts[::4, :] = -1
    count = 0
    for a in acts:
        env.act(a)
        count += int(env.observe()[2].sum())
    after = lookahead_info(env)
    assert count >= 5 * 16 and after["served"] == count and after["generated"] == 0, (count, after)
    assert enable_lookahead(env) == 0
    assert lookahead_info(env) == after, "a second call changes nothing"
    env.close()


def test_sixteen_game_list_sizes_slots_per_game(hostsim_lib):
    from level_lookahead import enable_lookahead, lookahead_info

    alone = _env(hostsim_lib, n=16, name="leaper")
    joint = _env(hostsim_lib, n=16, name="bigfish,bossfight,caveflyer,chaser,climber,coinrun,dodgeball,fruitbot,heist,jumper,"
                                          "leaper,maze,miner,ninja,plunder,starpilot")
    for env in (alone, joint):
        assert enable_lookahead(env) == 0
    # per env: one slot of its own game (24-77 KB) plus the list entry; staging at the handle's largest capacities
    assert lookahead_info(joint)["bytes"] > lookahead_info(alone)["bytes"]
    alone.close()
    joint.close()


HOST_CYCLES = r"""
import ctypes as C, gc, sys
sys.path.insert(0, {root!r}); sys.path.insert(0, {root!r} + "/tests")
libc = C.CDLL(None)
class Mallinfo2(C.Structure):
    _fields_ = [(k, C.c_size_t) for k in ("arena", "ordblks", "smblks", "hblks", "hblkhd", "usmblks", "fsmblks",
                                          "uordblks", "fordblks", "keepcost")]
libc.mallinfo2.restype = Mallinfo2
from level_bank import build_bank
from level_lookahead import enable_lookahead
from oracle.record import STANDIN_PACK
from oracle.ref_env import RefVecEnv, mt19937_actions

def cycle():
    env = RefVecEnv({num}, "coinrun", distribution_mode="easy", num_levels=0, rand_seed=0, lib_path={lib!r},
                    resource_root=STANDIN_PACK)
    assert build_bank(env, [1, 2, 3]) == 0
    assert enable_lookahead(env) == 0
    for actions in mt19937_actions(0, {num}, 3):
        actions[::7] = -1
        env.act(actions)
        env.observe()
    env.close()
    del env
    gc.collect()

def in_use():
    m = libc.mallinfo2()
    return m.uordblks + m.hblkhd

cycle()
before = in_use()
cycle()
cycle()
print("IN_USE", before, in_use())
"""


def test_close_returns_host_build_memory(hostsim_lib):
    """As tests/test_handle_lifetime.py, with lookahead on: the bytes in use do not grow across two cycles by as much
    as a byte per env."""
    if not hasattr(C.CDLL(None), "mallinfo2"):
        pytest.skip("glibc without mallinfo2")
    num = 1024
    env = dict(os.environ, GLIBC_TUNABLES="glibc.malloc.tcache_count=0")
    out = subprocess.run([sys.executable, "-c", HOST_CYCLES.format(root=ROOT, lib=hostsim_lib, num=num)],
                         env=env, capture_output=True, text=True)
    lines = [ln for ln in out.stdout.splitlines() if ln.startswith("IN_USE")]
    assert lines, out.stdout[-2000:] + out.stderr[-4000:]
    before, after = map(int, lines[0].split()[1:])
    assert after - before < num, f"two handles left {after - before} bytes of heap behind"
