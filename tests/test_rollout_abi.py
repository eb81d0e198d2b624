"""pgb200_get_rollout without a GPU: exported by both builds and declared by the header; in the host debug build, bad and
changed slot counts are refused, the first call stores the outputs current at the call into slot 0, a second call
returns the same pointers, and a closed handle gives back every byte the rollout took from the process's heap."""
import ctypes as C
import os
import re
import subprocess
import sys

import numpy as np
import pytest

from procgen_b200 import libenv as L

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "procgen_b200.h")


def _env(lib, n=16, name="coinrun", **kw):
    from oracle.ref_env import RefVecEnv, default_pack

    return RefVecEnv(n, name, **dict(dict(distribution_mode="hard", num_levels=0, rand_seed=0), **kw), resource_root=default_pack(), lib_path=lib)


def test_exported(product_lib, hostsim_lib):
    for path in (product_lib, hostsim_lib):
        assert hasattr(C.CDLL(path), "pgb200_get_rollout")
    assert "pgb200_get_rollout" in L.EXPORTS
    text = open(HEADER).read()
    assert re.search(r"LIBENV_API int pgb200_get_rollout\(libenv_env \*handle, int slots, struct pgb200_rollout \*out\);", text)
    assert [name for name, _ in L.Rollout._fields_] == ["rgb", "rew", "first", "cursor"]


def test_bad_and_changed_slots(hostsim_lib):
    from rollout import get_rollout

    env = _env(hostsim_lib)
    for slots in (-1, 0, 1):
        assert get_rollout(env, slots)[0] == -1
    rc, roll = get_rollout(env, 3)
    assert rc == 0
    for slots in (1, 2, 4):
        assert get_rollout(env, slots)[0] == -1, "a later call with another slot count"
    rc, again = get_rollout(env, 3)
    assert rc == 0 and again["pointers"] == roll["pointers"], "a later call with the same slots returns the same arrays"
    env.close()


def test_slot_zero_holds_the_outputs_of_the_first_call(hostsim_lib):
    from oracle.ref_env import mt19937_actions
    from rollout import get_rollout

    n = 16
    env = _env(hostsim_lib, n=n, name="bigfish,bossfight,caveflyer,chaser")
    for a in mt19937_actions(0, n, 30):
        a[::3] = -1  # resets by the caller: first is set for those envs
        env.act(a)
    rew, ob, first = env.observe()
    assert first.any(), "a step with first set, so that slot 0 is not just zeros"
    rc, roll = get_rollout(env, 5)
    assert rc == 0
    assert roll["cursor"][0] == 0
    assert np.array_equal(roll["rgb"][0], ob["rgb"]) and np.array_equal(roll["rew"][0], rew) and np.array_equal(roll["first"][0], first)
    assert not roll["rgb"][1:].any() and not roll["rew"][1:].any() and not roll["first"][1:].any()
    env.act(mt19937_actions(1, n, 1)[0])
    rew, ob, first = env.observe()
    assert roll["cursor"][0] == 1 and np.array_equal(roll["rgb"][1], ob["rgb"]) and np.array_equal(roll["rew"][1], rew)
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
from rollout import get_rollout

def cycle():
    env = RefVecEnv({num}, "coinrun", distribution_mode="easy", num_levels=0, rand_seed=0, lib_path={lib!r},
                    resource_root=STANDIN_PACK)
    rc, roll = get_rollout(env, 3)
    assert rc == 0
    del roll
    for actions in mt19937_actions(0, {num}, 4):
        env.act(actions)
        env.observe()
    env.close()
    del env
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
    """As tests/test_handle_lifetime.py, with the rollout on (36 KiB per env here): after two cycles, in which the
    interpreter's own caches settle, the bytes in use do not grow across three more by as much as a byte per env."""
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
