"""Snapshot slots (pgb200_get_snapshots / pgb200_apply_snapshots) on a libenv-ABI handle of the library under test
(oracle.ref_env.RefVecEnv), for the tests: the store's arrays, one apply, and an env's header and live entities as
pgb200_debug_read_env reads them."""
import ctypes as C

import numpy as np

from helpers import lib_array

HDR_BYTES, ENT_BYTES, MAX_ENTS = 512, 128, 1024


def _declare(lib):
    from procgen_b200.libenv import Snapshots

    lib.pgb200_get_snapshots.argtypes = [C.c_void_p, C.c_int, C.POINTER(Snapshots)]
    lib.pgb200_get_snapshots.restype = C.c_int
    lib.pgb200_apply_snapshots.argtypes = [C.c_void_p]
    lib.pgb200_apply_snapshots.restype = C.c_int
    lib.pgb200_debug_read_env.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int]
    lib.pgb200_debug_read_env.restype = C.c_int
    lib.pgb200_kernel_launches.argtypes = [C.c_void_p]
    lib.pgb200_kernel_launches.restype = C.c_int64


def get_snapshots(env, slots):
    """(pgb200_get_snapshots' result, {"save_from", "load_from", "source"} as helpers.lib_array, "pointers", "bytes"}, or
    None on -1)"""
    from procgen_b200.libenv import Snapshots

    _declare(env.lib)
    out = Snapshots()
    rc = env.lib.pgb200_get_snapshots(C.c_void_p(env.h), int(slots), C.byref(out))
    if rc != 0:
        return rc, None
    return rc, {"save_from": lib_array(env, out.save_from, (slots,), "<i4"),
                "load_from": lib_array(env, out.load_from, (env.num,), "<i4"),
                "source": lib_array(env, out.source, (slots,), "<i4"),
                "pointers": (out.save_from, out.load_from, out.source), "bytes": out.bytes}


def apply(env):
    _declare(env.lib)
    return env.lib.pgb200_apply_snapshots(C.c_void_p(env.h))


def launches(env):
    _declare(env.lib)
    return int(env.lib.pgb200_kernel_launches(C.c_void_p(env.h)))


def read_env(env, e):
    """(env e's header, its live entities) as bytes"""
    _declare(env.lib)
    hdr = (C.c_uint8 * HDR_BYTES)()
    ents = (C.c_uint8 * (ENT_BYTES * MAX_ENTS))()
    n = env.lib.pgb200_debug_read_env(C.c_void_p(env.h), int(e), hdr, ents, MAX_ENTS)
    assert 0 <= n <= MAX_ENTS, n
    return bytes(hdr), bytes(ents)[:n * ENT_BYTES]


def same_game(n, games, e, exclude=()):
    """The envs of env e's game (env i plays game i % games), without those in `exclude`"""
    return [i for i in range(e % games, n, games) if i not in exclude]


def observation(env):
    """{name: copy} of a RefVecEnv's rew, rgb, first and infos after libenv_observe"""
    rew, ob, first = env.observe()
    out = {"rew": np.array(rew), "rgb": np.array(ob["rgb"]), "first": np.array(first)}
    out.update({k: np.array(v) for k, v in env.info.items()})
    return out


def assert_same(a, b, envs, when):
    envs = np.asarray(envs, dtype=np.int64)
    for k in a:
        x, y = a[k][envs], b[k][envs]
        if not np.array_equal(x, y):
            bad = np.nonzero((x != y).reshape(len(envs), -1).any(1))[0]
            raise AssertionError(f"{when}: {k} differs at envs {envs[bad[:8]]}")
