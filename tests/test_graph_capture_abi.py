"""The CUDA-graph entry point of the C ABI without a GPU: exported by the product library, and the host debug build
(which has no device slot to hand out) refuses it."""
import ctypes as C

from procgen_b200 import libenv as L


def test_consumer_slot_device_exported(product_lib):
    lib = C.CDLL(product_lib)
    assert hasattr(lib, "pgb200_get_consumer_slot_device")
    assert "pgb200_get_consumer_slot_device" in L.EXPORTS


def test_consumer_slot_device_refused_by_host_build(hostsim_lib):
    from oracle.record import STANDIN_PACK
    from oracle.ref_env import RefVecEnv

    env = RefVecEnv(4, "coinrun", distribution_mode="easy", num_levels=0, rand_seed=0, lib_path=hostsim_lib, resource_root=STANDIN_PACK)
    lib = L.bind(C.CDLL(hostsim_lib))
    out = C.POINTER(C.c_int32)()
    assert lib.pgb200_get_consumer_slot_device(C.c_void_p(env.h), C.byref(out)) == -1
    assert not out
    # stepping, the consumer slot and the capture checks of the host build are unchanged by the device counter
    env.act([0, 1, 2, 3])
    env.observe()
    assert lib.pgb200_consumer_slot(C.c_void_p(env.h)) == 0
    env.close()
