"""Level bank (pgb200_build_level_bank) helpers for the tests: build a bank on a libenv-ABI handle, read what it holds,
and run a banked handle in lockstep with an unbanked one of the same configuration. A bank changes nothing but speed,
so the unbanked handle is an exact control: every output, every state blob and every error bit must be equal."""
import ctypes as C

import numpy as np

from helpers import assert_same_observation
from oracle.ref_env import mt19937_actions


def _declare(lib):
    lib.pgb200_build_level_bank.argtypes = [C.c_void_p, C.POINTER(C.c_int32), C.c_int, C.c_int]
    lib.pgb200_build_level_bank.restype = C.c_int
    lib.pgb200_level_bank_info.argtypes = [C.c_void_p, C.POINTER(C.c_int), C.POINTER(C.c_int64)]
    lib.pgb200_level_bank_info.restype = C.c_int


def build_bank(env, seeds, capacity=0):
    """pgb200_build_level_bank on env (a RefVecEnv of the library); returns its result."""
    _declare(env.lib)
    arr = np.ascontiguousarray(np.asarray(list(seeds), np.int64).astype(np.int32))
    return env.lib.pgb200_build_level_bank(C.c_void_p(env.h), arr.ctypes.data_as(C.POINTER(C.c_int32)), int(arr.size), int(capacity))


def bank_info(env):
    """(distinct seeds banked, device bytes held)"""
    _declare(env.lib)
    levels, nbytes = C.c_int(-1), C.c_int64(-1)
    assert env.lib.pgb200_level_bank_info(C.c_void_p(env.h), C.byref(levels), C.byref(nbytes)) == 0
    return levels.value, nbytes.value


def error_bits(env):
    out = np.zeros(env.num, np.uint32)
    env.lib.pgb200_get_errors.restype = C.c_uint32
    env.lib.pgb200_get_errors(C.c_void_p(env.h), out.ctypes.data_as(C.POINTER(C.c_uint32)))
    return out


def force_resets(seed, every):
    """plan(t, actions): about one action in `every` becomes -1 (a reset by the caller)"""
    rs = np.random.RandomState(seed)

    def plan(t, actions):
        actions[rs.randint(every, size=len(actions)) == 0] = -1

    return plan


def run_bank_lockstep(ctrl, banked, steps, plan=None, action_seed=0, blob_every=25, check_errors=True):
    """ctrl and banked stepped together with mt19937 actions (plan(t, actions) may change them in place). Every step:
    equal outputs, and equal state blobs for every env that started a new episode; all blobs every `blob_every`
    steps and at the end; equal per-env error bits at the end. Returns the number of episode starts seen."""
    n = ctrl.num
    acts = mt19937_actions(action_seed, n, steps)
    assert_same_observation(ctrl, banked, -1)
    starts = 0
    for t in range(steps):
        a = acts[t].copy()
        if plan:
            plan(t, a)
        ctrl.act(a)
        banked.act(a)
        assert_same_observation(ctrl, banked, t)
        first = ctrl.first.copy()
        starts += int(first.sum())
        envs = range(n) if t % blob_every == 0 else np.nonzero(first)[0]
        for e in envs:
            assert ctrl.get_state(int(e)) == banked.get_state(int(e)), f"step {t} env {e}: state blobs differ"
    for e in range(n):
        assert ctrl.get_state(e) == banked.get_state(e), f"env {e}: state blobs differ at the end"
    if check_errors:
        ec, eb = error_bits(ctrl), error_bits(banked)
        assert np.array_equal(ec, eb), f"error bits differ at envs {np.nonzero(ec != eb)[0][:8]}"
    return starts
