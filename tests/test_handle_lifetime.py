"""A handle returns everything it allocated when it closes, with every opt-in device array turned on, in the host debug
build (the process's heap, counted by glibc) and on the GPU (the process's device memory, counted by NVML); and
pgb200_debug_read_env refuses an env index outside the handle."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NUM = 4096  # the smallest array of such a handle is one byte per env: the pause mask, 4 KiB

# One cycle makes a coinrun handle, turns on next-level seeds, final outputs, the pause mask and a level bank, steps it
# and closes it. The first cycle is a warm-up: the host build keeps one frame per thread for good (render_env_serial).
# The count is every byte malloc has handed out and not taken back, in the heap (uordblks) and in mappings of their
# own (hblkhd): a freed heap region may serve a large request, so mappings alone can miss a leak. It runs in a process
# of its own with malloc's per-thread cache off, whose chunks count as in use and would add a few KiB of noise.
HOST_CYCLES = r"""
import ctypes as C, gc, sys
sys.path.insert(0, {root!r}); sys.path.insert(0, {root!r} + "/tests")
libc = C.CDLL(None)
class Mallinfo2(C.Structure):
    _fields_ = [(k, C.c_size_t) for k in ("arena", "ordblks", "smblks", "hblks", "hblkhd", "usmblks", "fsmblks",
                                          "uordblks", "fordblks", "keepcost")]
libc.mallinfo2.restype = Mallinfo2
from final_obs_oracle import LibFinal
from level_bank import build_bank
from level_seed_oracle import next_level_seeds
from oracle.record import STANDIN_PACK
from oracle.ref_env import RefVecEnv, mt19937_actions
from pause_oracle import pause_mask

def cycle():
    env = RefVecEnv({num}, "coinrun", distribution_mode="easy", num_levels=0, rand_seed=0, lib_path={lib!r},
                    resource_root=STANDIN_PACK)
    next_level_seeds(env)
    LibFinal(env)
    pause_mask(env)[::2] = 1
    assert build_bank(env, [1, 2, 3]) == 0
    for actions in mt19937_actions(0, {num}, 3):
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
    """The bytes in use do not grow across two cycles by as much as the handle's smallest array."""
    if not hasattr(C.CDLL(None), "mallinfo2"):
        pytest.skip("glibc without mallinfo2")
    env = dict(os.environ, GLIBC_TUNABLES="glibc.malloc.tcache_count=0")
    out = subprocess.run([sys.executable, "-c", HOST_CYCLES.format(root=ROOT, lib=hostsim_lib, num=NUM)],
                         env=env, capture_output=True, text=True)
    lines = [ln for ln in out.stdout.splitlines() if ln.startswith("IN_USE")]
    assert lines, out.stdout[-2000:] + out.stderr[-4000:]
    before, after = map(int, lines[0].split()[1:])
    assert after - before < NUM, f"two handles left {after - before} bytes of heap behind"


def test_debug_read_env_refuses_out_of_range(hostsim_lib):
    from oracle.record import STANDIN_PACK
    from oracle.ref_env import RefVecEnv

    env = RefVecEnv(4, "coinrun", distribution_mode="easy", lib_path=hostsim_lib, resource_root=STANDIN_PACK)
    lib = env.lib
    lib.pgb200_debug_read_env.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int]
    lib.pgb200_debug_read_env.restype = C.c_int
    hdr = np.zeros(4096, np.uint8)
    ents = np.zeros(4096, np.uint8)
    for e in (-1, env.num):
        assert lib.pgb200_debug_read_env(env.h, e, hdr.ctypes.data, ents.ctypes.data, 1) == -1, f"env {e}"
        assert not hdr.any() and not ents.any(), f"env {e}: something was copied"
    assert lib.pgb200_debug_read_env(env.h, env.num - 1, hdr.ctypes.data, None, 0) > 0
    assert hdr.any()
    env.close()


def _process_device_bytes(pynvml):
    """This process's device memory on every GPU NVML lists it on, or None where NVML does not show it."""
    pid, total, seen = os.getpid(), 0, False
    for i in range(pynvml.nvmlDeviceGetCount()):
        for proc in pynvml.nvmlDeviceGetComputeRunningProcesses(pynvml.nvmlDeviceGetHandleByIndex(i)):
            if proc.pid == pid and proc.usedGpuMemory is not None:
                total += proc.usedGpuMemory
                seen = True
    return total if seen else None


@pytest.mark.gpu
def test_close_returns_device_memory(product_lib):
    """The device-resident twin, with the consumer output on as well: the process's device memory does not grow across
    two cycles by a 2 MiB page, the unit NVML counts in. The machine may run other work, hence per process."""
    pynvml = pytest.importorskip("pynvml")
    import torch

    from oracle.record import STANDIN_PACK
    from oracle.ref_env import mt19937_actions
    from procgen_b200 import ProcgenGym3Env

    def cycle():
        env = ProcgenGym3Env(NUM, "coinrun", distribution_mode="easy", num_levels=0, rand_seed=0, resource_root=STANDIN_PACK)
        env.next_level_seeds()
        env.final_outputs()
        env.pause_mask()[::2] = 1
        env.build_level_bank([1, 2, 3])
        env.enable_consumer_output(torch.float16, 2)
        for actions in mt19937_actions(0, NUM, 3):
            env.act(torch.as_tensor(actions, device="cuda"))
            env.consumer_observation()
        env.close()
        del env
        torch.cuda.synchronize()
        torch.cuda.empty_cache()

    pynvml.nvmlInit()
    try:
        cycle()
        before = _process_device_bytes(pynvml)
        if before is None:
            pytest.skip("NVML does not list this process (PID namespace)")
        cycle()
        cycle()
        after = _process_device_bytes(pynvml)
    finally:
        pynvml.nvmlShutdown()
    assert after - before < 2 << 20, f"two handles left {after - before} bytes of device memory behind"
