"""Level lookahead (pgb200_enable_level_lookahead) helpers for the tests: turn it on for a libenv-ABI handle, read its
counters, and count the resets a lockstep run makes. Lookahead changes nothing but speed, so a handle without it is an
exact control (level_bank.run_bank_lockstep compares every output, state blob and error bit); the counters are what
shows that the resets were served from the slots at all."""
import ctypes as C

import numpy as np

from helpers import assert_same_observation
from level_bank import error_bits
from oracle.ref_env import mt19937_actions


def _declare(lib):
    lib.pgb200_enable_level_lookahead.argtypes = [C.c_void_p]
    lib.pgb200_enable_level_lookahead.restype = C.c_int
    lib.pgb200_level_lookahead_info.argtypes = [C.c_void_p, C.POINTER(C.c_int64)]
    lib.pgb200_level_lookahead_info.restype = C.c_int


def enable_lookahead(env):
    """pgb200_enable_level_lookahead on env (a RefVecEnv of the library); returns its result."""
    _declare(env.lib)
    return env.lib.pgb200_enable_level_lookahead(C.c_void_p(env.h))


def lookahead_info(env):
    """{"served": resets served from a slot, "bank": from the bank, "generated": resets that generated, "bytes": held}"""
    _declare(env.lib)
    out = (C.c_int64 * 4)(-1, -1, -1, -1)
    assert env.lib.pgb200_level_lookahead_info(C.c_void_p(env.h), out) == 0
    return dict(zip(("served", "bank", "generated", "bytes"), list(out)))


def resets(info):
    return info["served"] + info["bank"] + info["generated"]


def run_counted_lockstep(ref, dut, steps, plan=None, action_seed=0, blob_every=25, sequential=False, check_errors=True):
    """ref (a handle without lookahead, or the oracle) and dut (lookahead on) stepped together with mt19937 actions
    (plan(t, actions) may change them in place). Every step: equal outputs, equal state blobs for every env that reset,
    all blobs every `blob_every` steps and at the end, and (check_errors) equal error bits at the end. Returns the
    resets dut made: every `first`, and under use_sequential_levels (`sequential`) also the completed levels, which go
    on with first = 0. Each must be counted once by dut's counters."""
    n = ref.num
    acts = mt19937_actions(action_seed, n, steps)
    assert_same_observation(ref, dut, -1)
    before = resets(lookahead_info(dut))
    count = 0
    for t in range(steps):
        a = acts[t].copy()
        if plan:
            plan(t, a)
        ref.act(a)
        dut.act(a)
        assert_same_observation(ref, dut, t)
        reset = ref.first.astype(bool).copy()
        if sequential:
            reset |= ref.info["prev_level_complete"].astype(bool)
        count += int(reset.sum())
        envs = range(n) if t % blob_every == 0 else np.nonzero(reset)[0]
        for e in envs:
            assert ref.get_state(int(e)) == dut.get_state(int(e)), f"step {t} env {e}: state blobs differ"
    for e in range(n):
        assert ref.get_state(e) == dut.get_state(e), f"env {e}: state blobs differ at the end"
    if check_errors:
        er, ed = error_bits(ref), error_bits(dut)
        assert np.array_equal(er, ed), f"error bits differ at envs {np.nonzero(er != ed)[0][:8]}"
    assert resets(lookahead_info(dut)) - before == count, f"{count} resets, counters {lookahead_info(dut)}"
    return count
