"""The action-repeat entry point of the C ABI: exported by both builds and declared by the header; in the host debug
build every count is 1 at the first call, a later call returns the same array, and a closed handle gives back every
byte the array took from the process's heap. On the GPU, the first call is refused while the handle's stream captures."""
import ctypes as C
import os
import re
import subprocess
import sys

import pytest

from procgen_b200 import libenv as L

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "procgen_b200.h")


def test_exported(product_lib, hostsim_lib):
    for path in (product_lib, hostsim_lib):
        assert hasattr(C.CDLL(path), "pgb200_get_action_repeat")
    assert "pgb200_get_action_repeat" in L.EXPORTS
    assert re.search(r"LIBENV_API int pgb200_get_action_repeat\(libenv_env \*handle, int32_t \*\*out\);", open(HEADER).read())


def test_ones_at_the_first_call_and_the_same_array_again(hostsim_lib):
    import numpy as np

    from action_repeat_oracle import action_repeat
    from oracle.record import STANDIN_PACK
    from oracle.ref_env import RefVecEnv

    env = RefVecEnv(38, "coinrun,maze", distribution_mode="hard", num_levels=0, rand_seed=0, resource_root=STANDIN_PACK,
                    lib_path=hostsim_lib)
    rep = action_repeat(env)
    assert rep.dtype == np.int32 and rep.shape == (38,) and (rep == 1).all()
    rep[:] = np.arange(38)
    again = action_repeat(env)
    assert again.ctypes.data == rep.ctypes.data and (again == np.arange(38)).all(), "a later call allocates nothing"
    env.act(np.zeros(38, np.int32))
    assert (rep == np.arange(38)).all(), "a step leaves the counts as they are"
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
from action_repeat_oracle import action_repeat

def cycle():
    env = RefVecEnv({num}, "coinrun", distribution_mode="easy", num_levels=0, rand_seed=0, lib_path={lib!r},
                    resource_root=STANDIN_PACK)
    rep = action_repeat(env)
    rep[:] = 3
    for actions in mt19937_actions(0, {num}, 2):
        env.act(actions)
    env.close()
    del env, rep
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
    """As tests/test_rollout_abi.py: the bytes in use do not grow across three more cycles by as much as a byte per
    env (the counts alone take four per env)."""
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


@pytest.mark.gpu
def test_first_call_refused_under_capture(product_lib):
    """The first call allocates and waits for the device: with the handle's stream capturing it returns -1 and hands
    out nothing. Once the array exists, a call under capture returns it."""
    import torch

    from oracle.record import STANDIN_PACK
    from procgen_b200 import ProcgenGym3Env

    env = ProcgenGym3Env(64, "coinrun", distribution_mode="easy", num_levels=0, rand_seed=0, resource_root=STANDIN_PACK)
    lib = env._lib
    side = torch.cuda.Stream()
    out = C.POINTER(C.c_int32)()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=side):
        lib.pgb200_set_stream(env._h, C.c_void_p(side.cuda_stream))
        rc = lib.pgb200_get_action_repeat(env._h, C.byref(out))
        torch.zeros(1, device="cuda").add_(1)
    assert rc == -1 and not out
    rep = env.action_repeat()
    with torch.cuda.graph(torch.cuda.CUDAGraph(), stream=side):
        lib.pgb200_set_stream(env._h, C.c_void_p(side.cuda_stream))
        rc = lib.pgb200_get_action_repeat(env._h, C.byref(out))
        torch.zeros(1, device="cuda").add_(1)
    assert rc == 0 and C.cast(out, C.c_void_p).value == rep.data_ptr()
    env._stream_handle = side.cuda_stream
    assert env.errors() == 0
    env.close()
