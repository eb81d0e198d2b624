"""pgb200_get_snapshots / pgb200_apply_snapshots without a GPU: exported by both builds and declared by the header; in the
host debug build, refused `slots` values change nothing, a later call returns the same arrays, an apply needs a store,
and a closed handle gives back every byte its store took from the process's heap."""
import ctypes as C
import os
import re
import subprocess
import sys

import pytest

from procgen_b200 import libenv as L
from snapshots import apply, get_snapshots

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "procgen_b200.h")


def _env(lib, n=8, name="coinrun", **kw):
    from oracle.ref_env import RefVecEnv, default_pack

    return RefVecEnv(n, name, **dict(dict(distribution_mode="hard", num_levels=0, rand_seed=0), **kw), resource_root=default_pack(), lib_path=lib)


def test_exported(product_lib, hostsim_lib):
    for path in (product_lib, hostsim_lib):
        lib = C.CDLL(path)
        assert hasattr(lib, "pgb200_get_snapshots") and hasattr(lib, "pgb200_apply_snapshots")
    assert {"pgb200_get_snapshots", "pgb200_apply_snapshots"} <= set(L.EXPORTS)
    text = open(HEADER).read()
    assert re.search(r"LIBENV_API int pgb200_get_snapshots\(libenv_env \*handle, int slots, struct pgb200_snapshots \*out\);", text)
    assert re.search(r"LIBENV_API int pgb200_apply_snapshots\(libenv_env \*handle\);", text)
    fields = re.search(r"struct pgb200_snapshots \{(.*?)\};", text, re.S).group(1)
    assert [ln.split("/*")[0].split()[-1].strip(";*") for ln in fields.strip().splitlines()] == [
        name for name, _ in L.Snapshots._fields_]


def test_store_arguments(hostsim_lib):
    env = _env(hostsim_lib)
    assert apply(env) == -1, "an apply without a store"
    before = [env.get_state(e) for e in range(env.num)]
    for bad in (0, -1, -100):
        assert get_snapshots(env, bad)[0] == -1, bad
    # a store this build cannot allocate: about 2^31 slots of tens of kilobytes
    assert get_snapshots(env, 2 ** 31 - 1)[0] == -1
    assert apply(env) == -1
    rc, st = get_snapshots(env, 5)
    assert rc == 0
    assert (st["save_from"] == -1).all() and (st["source"] == -1).all() and (st["load_from"] == -1).all()
    assert st["bytes"] > 5 * 16 * 1024, st["bytes"]
    rc, again = get_snapshots(env, 5)
    assert rc == 0 and again["pointers"] == st["pointers"] and again["bytes"] == st["bytes"]
    for other in (4, 6, 0):
        assert get_snapshots(env, other)[0] == -1, other
    assert [env.get_state(e) for e in range(env.num)] == before, "the store changed an env"
    # an apply with every entry -1 changes nothing either
    assert apply(env) == 0
    assert [env.get_state(e) for e in range(env.num)] == before
    env.close()


def _slot_bytes(lib, name):
    """The bytes one more slot of a store costs on a handle of `name`"""
    total = []
    for slots in (1, 3):
        env = _env(lib, n=2, name=name)
        rc, st = get_snapshots(env, slots)
        env.close()
        assert rc == 0
        total.append(st["bytes"])
    return (total[1] - total[0]) // 2


def test_slot_size_follows_the_strides(hostsim_lib):
    """Every slot is sized for the largest live state of the list"""
    sizes = {name: _slot_bytes(hostsim_lib, name) for name in ("coinrun", "maze", "coinrun,maze")}
    assert sizes["coinrun,maze"] >= max(sizes["coinrun"], sizes["maze"]), sizes


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
from snapshots import apply, get_snapshots

def cycle():
    env = RefVecEnv({num}, "coinrun", distribution_mode="easy", num_levels=0, rand_seed=0, lib_path={lib!r},
                    resource_root=STANDIN_PACK)
    rc, st = get_snapshots(env, 64)
    assert rc == 0
    st["save_from"][:] = range(64)
    st["load_from"][:64] = range(63, -1, -1)
    assert apply(env) == 0
    for actions in mt19937_actions(0, {num}, 3):
        env.act(actions)
    env.close()
    del env, st
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
    """As tests/test_rollout_abi.py, with a 64-slot store, saves and loads in each cycle: the bytes in use do not grow
    across three more cycles by as much as a byte per env."""
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
