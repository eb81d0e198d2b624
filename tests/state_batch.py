"""pgb200_get_states / pgb200_set_states on a libenv-ABI handle of the library under test (oracle.ref_env.RefVecEnv),
for the tests: the batched calls, and the subsets they are tried on."""
import ctypes as C

import numpy as np


def _declare(lib):
    lib.pgb200_get_states.argtypes = [C.c_void_p, C.POINTER(C.c_int32), C.c_int, C.POINTER(C.c_void_p), C.POINTER(C.POINTER(C.c_int64))]
    lib.pgb200_get_states.restype = C.c_int
    lib.pgb200_set_states.argtypes = [C.c_void_p, C.POINTER(C.c_int32), C.c_int, C.c_char_p, C.POINTER(C.c_int64)]
    lib.pgb200_set_states.restype = C.c_int


def get_states_raw(env, envs, n=None):
    """(the call's result, the data address, the offsets as a list) of pgb200_get_states of `envs` (n entries)"""
    _declare(env.lib)
    arr = np.ascontiguousarray(np.asarray(envs, np.int32).reshape(-1))
    data, offsets = C.c_void_p(), C.POINTER(C.c_int64)()
    n = arr.size if n is None else n
    rc = env.lib.pgb200_get_states(C.c_void_p(env.h), arr.ctypes.data_as(C.POINTER(C.c_int32)), int(n), C.byref(data), C.byref(offsets))
    if rc != 0:
        return rc, None, None
    return rc, data.value, np.ctypeslib.as_array(offsets, shape=(max(n, 0) + 1,)).tolist()


def get_states(env, envs):
    """The blobs of envs, in order, from one pgb200_get_states"""
    rc, data, offs = get_states_raw(env, envs)
    assert rc == 0
    return [C.string_at(data + offs[i], offs[i + 1] - offs[i]) for i in range(len(offs) - 1)]


def set_states(env, envs, blobs, n=None):
    """pgb200_set_states of blobs into envs; returns its result"""
    _declare(env.lib)
    arr = np.ascontiguousarray(np.asarray(envs, np.int32).reshape(-1))
    offsets = np.zeros(len(blobs) + 1, np.int64)
    offsets[1:] = np.cumsum([len(b) for b in blobs])
    n = arr.size if n is None else n
    return env.lib.pgb200_set_states(C.c_void_p(env.h), arr.ctypes.data_as(C.POINTER(C.c_int32)), int(n), b"".join(blobs),
                                     offsets.ctypes.data_as(C.POINTER(C.c_int64)))


def subset_with_duplicates(rng, n, size):
    """size random env indices of [0, n), unsorted, with at least one repeated"""
    s = list(rng.randint(0, n, size=size - 1))
    s.insert(int(rng.randint(0, size)), s[0])
    return [int(e) for e in s]


def distinct_subset(rng, n, size):
    """size distinct env indices of [0, n), unsorted"""
    return [int(e) for e in rng.permutation(n)[:size]]
