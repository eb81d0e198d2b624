"""pgb200_get_states / pgb200_set_states without a GPU: exported by both builds and declared by the header; in the host
debug build, refused arguments change nothing, an empty list works, the blobs pgb200_get_states hands out stay where
they are until its next call, and a closed handle gives back every byte the transfers took from the process's heap."""
import ctypes as C
import os
import re
import subprocess
import sys

import pytest

from procgen_b200 import libenv as L
from state_batch import get_states, get_states_raw, set_states

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "procgen_b200.h")


def _env(lib, n=8, name="coinrun", **kw):
    from oracle.ref_env import RefVecEnv, default_pack

    return RefVecEnv(n, name, **dict(dict(distribution_mode="hard", num_levels=0, rand_seed=0), **kw), resource_root=default_pack(), lib_path=lib)


def test_exported(product_lib, hostsim_lib):
    for path in (product_lib, hostsim_lib):
        lib = C.CDLL(path)
        assert hasattr(lib, "pgb200_get_states") and hasattr(lib, "pgb200_set_states")
    assert {"pgb200_get_states", "pgb200_set_states"} <= set(L.EXPORTS)
    text = open(HEADER).read()
    assert re.search(r"LIBENV_API int pgb200_get_states\(libenv_env \*handle, const int32_t \*envs, int n, const char \*\*data, "
                     r"const int64_t \*\*offsets\);", text)
    assert re.search(r"LIBENV_API int pgb200_set_states\(libenv_env \*handle, const int32_t \*envs, int n, const char \*data, "
                     r"const int64_t \*offsets\);", text)


def test_refused_arguments_change_nothing(hostsim_lib):
    from oracle.ref_env import mt19937_actions

    env = _env(hostsim_lib)
    for a in mt19937_actions(0, env.num, 10):
        env.act(a)
    before = [env.get_state(e) for e in range(env.num)]
    other = _env(hostsim_lib, rand_seed=3)
    blobs = [other.get_state(e) for e in range(env.num)]
    assert get_states_raw(env, [0], n=-1)[0] == -1
    for bad in ([0, env.num], [-1], [3, 2, env.num + 5]):
        assert get_states_raw(env, bad)[0] == -1, bad
        assert set_states(env, bad, blobs[:len(bad)]) == -1, bad
    assert set_states(env, [0], blobs[:1], n=-1) == -1
    assert set_states(env, [1, 4, 1], blobs[:3]) == -1, "an env listed twice"
    assert [env.get_state(e) for e in range(env.num)] == before
    # an accepted call then does what it should
    assert set_states(env, [4, 1], [blobs[4], blobs[1]]) == 0
    assert get_states(env, [1, 4]) == [blobs[1], blobs[4]]
    env.close()
    other.close()


def test_empty_list(hostsim_lib):
    env = _env(hostsim_lib)
    before = [env.get_state(e) for e in range(env.num)]
    rc, _, offs = get_states_raw(env, [])
    assert rc == 0 and offs == [0]
    assert set_states(env, [], []) == 0
    assert [env.get_state(e) for e in range(env.num)] == before
    env.close()


def test_blobs_stay_until_the_next_call(hostsim_lib):
    """The arrays pgb200_get_states hands out keep their place and bytes across steps and get_state / set_state, and
    duplicates give the same blob twice"""
    from oracle.ref_env import mt19937_actions

    env = _env(hostsim_lib)
    envs = [5, 2, 5, 7]
    rc, data, offs = get_states_raw(env, envs)
    assert rc == 0
    raw = C.string_at(data, offs[-1])
    assert raw[offs[0]:offs[1]] == raw[offs[2]:offs[3]] == env.get_state(5)
    for a in mt19937_actions(1, env.num, 5):
        env.act(a)
    env.set_state(2, env.get_state(3))
    assert C.string_at(data, offs[-1]) == raw
    rc, data2, offs2 = get_states_raw(env, [0])
    assert rc == 0 and C.string_at(data2, offs2[-1]) == env.get_state(0)
    env.close()


HOST_CYCLES = r"""
import ctypes as C, gc, sys
sys.path.insert(0, {root!r}); sys.path.insert(0, {root!r} + "/tests")
libc = C.CDLL(None)
class Mallinfo2(C.Structure):
    _fields_ = [(k, C.c_size_t) for k in ("arena", "ordblks", "smblks", "hblks", "hblkhd", "usmblks", "fsmblks",
                                          "uordblks", "fordblks", "keepcost")]
libc.mallinfo2.restype = Mallinfo2
from oracle.record import STANDIN_PACK
from oracle.ref_env import RefVecEnv, mt19937_actions
from state_batch import get_states, set_states

def cycle():
    env = RefVecEnv({num}, "coinrun", distribution_mode="easy", num_levels=0, rand_seed=0, lib_path={lib!r},
                    resource_root=STANDIN_PACK)
    for actions in mt19937_actions(0, {num}, 3):
        env.act(actions)
    blobs = get_states(env, list(range({num})))
    assert set_states(env, list(range({num}))[::-1], blobs[::-1]) == 0
    env.close()
    del env, blobs
    gc.collect()

def in_use():
    m = libc.mallinfo2()
    return m.uordblks + m.hblkhd

cycle()
cycle()
before = in_use()
cycle()
cycle()
cycle()
print("IN_USE", before, in_use())
"""


def test_close_returns_host_build_memory(hostsim_lib):
    """As tests/test_rollout_abi.py, with a get_states and a set_states of every env in each cycle: the bytes in use
    do not grow across three more cycles by as much as a byte per env."""
    if not hasattr(C.CDLL(None), "mallinfo2"):
        pytest.skip("glibc without mallinfo2")
    num = 1024
    env = dict(os.environ, GLIBC_TUNABLES="glibc.malloc.tcache_count=0")
    out = subprocess.run([sys.executable, "-c", HOST_CYCLES.format(root=ROOT, lib=hostsim_lib, num=num)],
                         env=env, capture_output=True, text=True)
    lines = [ln for ln in out.stdout.splitlines() if ln.startswith("IN_USE")]
    assert lines, out.stdout[-2000:] + out.stderr[-4000:]
    before, after = map(int, lines[0].split()[1:])
    assert after - before < num, f"three handles left {after - before} bytes of heap behind"
