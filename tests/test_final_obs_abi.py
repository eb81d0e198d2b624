"""The final-outputs entry point of the C ABI without a GPU: exported by both builds, its header constants and struct
restated by procgen_b200.libenv, and the rules of the first call and of set_state in the host debug build."""
import ctypes as C
import os
import re

import numpy as np

from procgen_b200 import libenv as L

HEADER = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "procgen_b200.h")


def test_exported(product_lib, hostsim_lib):
    for path in (product_lib, hostsim_lib):
        assert hasattr(C.CDLL(path), "pgb200_get_final_outputs")
    assert "pgb200_get_final_outputs" in L.EXPORTS


def test_header_constants_and_struct():
    text = open(HEADER).read()
    consts = {k: int(v) for k, v in re.findall(r"#define PGB200_LEVEL_END_(\w+) (\d+)", text)}
    assert consts == {"GAME": L.LEVEL_END_GAME, "TIMEOUT": L.LEVEL_END_TIMEOUT, "CALLER": L.LEVEL_END_CALLER} == {"GAME": 1, "TIMEOUT": 2, "CALLER": 3}
    body = re.search(r"struct pgb200_final_outputs \{(.*?)\};", text, re.S).group(1)
    assert re.findall(r"uint8_t \*(\w+);", body) == [f[0] for f in L.FinalOutputs._fields_] == ["rgb", "level_end"]
    assert re.search(r"LIBENV_API int pgb200_get_final_outputs\(libenv_env \*handle, struct pgb200_final_outputs \*out\);", text)


def test_first_call_and_set_state(hostsim_lib):
    """The first call returns zero-filled arrays after the initial reset, later calls the same arrays; set_state
    writes nothing to them."""
    from final_obs_oracle import LibFinal
    from oracle.record import STANDIN_PACK
    from oracle.ref_env import RefVecEnv

    kw = dict(distribution_mode="easy", num_levels=0, rand_seed=0, resource_root=STANDIN_PACK)
    env = RefVecEnv(4, "coinrun", lib_path=hostsim_lib, **kw)
    donor = RefVecEnv(4, "coinrun", lib_path=hostsim_lib, **dict(kw, rand_seed=3))
    fin = LibFinal(env)
    le, rgb = fin.read()
    assert not le.any() and not rgb.any()
    env.act(np.array([-1, -1, 0, 0], np.int32))
    env.observe()
    le, rgb = fin.read()
    assert le.tolist() == [3, 3, 0, 0] and rgb[:2].any() and not rgb[2:].any()
    for e in range(4):
        env.set_state(e, donor.get_state(e))
    le2, rgb2 = LibFinal(env).read()
    assert np.array_equal(le, le2) and np.array_equal(rgb, rgb2)
    env.close()
    donor.close()
