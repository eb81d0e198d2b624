"""The pause-mask entry point of the C ABI without a GPU: exported by both builds and declared by the header, and in
the host debug build a zero-filled mask gives the outputs and states of a handle without one."""
import ctypes as C
import os
import re

import numpy as np

from procgen_b200 import libenv as L

HEADER = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "procgen_b200.h")
ALL16 = "bigfish,bossfight,caveflyer,chaser,climber,coinrun,dodgeball,fruitbot,heist,jumper,leaper,maze,miner,ninja,plunder,starpilot"


def test_exported(product_lib, hostsim_lib):
    for path in (product_lib, hostsim_lib):
        assert hasattr(C.CDLL(path), "pgb200_get_pause_mask")
    assert "pgb200_get_pause_mask" in L.EXPORTS
    assert re.search(r"LIBENV_API int pgb200_get_pause_mask\(libenv_env \*handle, uint8_t \*\*out\);", open(HEADER).read())


def test_zero_mask_equals_no_mask(hostsim_lib):
    """Two handles on the same seeds, one with a zero-filled mask requested before its first step: every step their
    outputs and state blobs are equal, and the mask is the same array on every call."""
    from helpers import assert_same_observation
    from oracle.record import STANDIN_PACK
    from oracle.ref_env import RefVecEnv, mt19937_actions
    from pause_oracle import pause_mask

    kw = dict(distribution_mode="hard", num_levels=0, rand_seed=0, resource_root=STANDIN_PACK, lib_path=hostsim_lib)
    plain = RefVecEnv(32, ALL16, **kw)
    masked = RefVecEnv(32, ALL16, **kw)
    mask = pause_mask(masked)
    assert mask.dtype == np.uint8 and mask.shape == (32,) and not mask.any()
    assert pause_mask(masked).ctypes.data == mask.ctypes.data
    acts = mt19937_actions(1, 32, 100)
    acts[np.random.RandomState(2).randint(16, size=acts.shape) == 0] = -1
    for t in range(100):
        plain.act(acts[t])
        masked.act(acts[t])
        assert_same_observation(plain, masked, t)
        if t % 20 == 0:
            for e in range(32):
                assert plain.get_state(e) == masked.get_state(e), f"step {t} env {e}"
    assert not mask.any()
    plain.close()
    masked.close()
