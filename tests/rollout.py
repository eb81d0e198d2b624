"""Rollout (pgb200_get_rollout) helpers for the tests: request it on a libenv-ABI handle of the library under test, and
check its invariant after every step. The rollout changes no output, so a handle without it is an exact control; what
the rollout itself must hold is a copy of the outputs: after every step the cursor has moved on by one slot, that slot
holds the step's rgb, rew and first byte for byte, and every other slot is as it was."""
import ctypes as C

import numpy as np

from helpers import assert_same_observation, lib_array, read_lib_array
from level_bank import error_bits
from oracle.ref_env import mt19937_actions

FRAME = (64, 64, 3)


def get_rollout(env, slots):
    """(pgb200_get_rollout's result, {"rgb", "rew", "first", "cursor"} as helpers.lib_array, or None on -1)"""
    from procgen_b200.libenv import Rollout

    lib = env.lib
    lib.pgb200_get_rollout.argtypes = [C.c_void_p, C.c_int, C.POINTER(Rollout)]
    lib.pgb200_get_rollout.restype = C.c_int
    out = Rollout()
    rc = lib.pgb200_get_rollout(C.c_void_p(env.h), int(slots), C.byref(out))
    if rc != 0:
        return rc, None
    n = env.num
    return rc, {"rgb": lib_array(env, out.rgb, (slots, n) + FRAME, "|u1"), "rew": lib_array(env, out.rew, (slots, n), "<f4"),
                "first": lib_array(env, out.first, (slots, n), "|u1"), "cursor": lib_array(env, out.cursor, (1,), "<i4"),
                "pointers": (out.rgb, out.rew, out.first, out.cursor)}


def snapshot(roll):
    return {k: read_lib_array(roll[k]) for k in ("rgb", "rew", "first", "cursor")}


class RolloutCheck:
    """The rollout of `env`, requested here with `slots` slots; check(t, rew, rgb, first) after each step of env."""

    def __init__(self, env, slots):
        rc, self.roll = get_rollout(env, slots)
        assert rc == 0
        self.slots = slots
        self.prev = snapshot(self.roll)
        rew, ob, first = env.observe()
        assert self.prev["cursor"][0] == 0
        self._assert_slot(0, rew, ob["rgb"], first, "the first call")

    def _assert_slot(self, c, rew, rgb, first, when):
        now = self.prev
        if not np.array_equal(now["rgb"][c], rgb):
            bad = np.nonzero((now["rgb"][c] != rgb).reshape(len(rgb), -1).any(1))[0]
            raise AssertionError(f"{when}: slot {c} rgb differs at envs {bad[:8]}")
        assert np.array_equal(now["rew"][c], rew), f"{when}: slot {c} rew differs at envs {np.nonzero(now['rew'][c] != rew)[0][:8]}"
        assert np.array_equal(now["first"][c], first), f"{when}: slot {c} first differs"

    def check(self, t, rew, rgb, first):
        before = self.prev
        self.prev = snapshot(self.roll)
        c = int(self.prev["cursor"][0])
        assert c == (int(before["cursor"][0]) + 1) % self.slots, f"step {t}: cursor {before['cursor'][0]} -> {c}"
        self._assert_slot(c, rew, rgb, first, f"step {t}")
        others = np.arange(self.slots) != c
        for k in ("rgb", "rew", "first"):
            assert np.array_equal(self.prev[k][others], before[k][others]), f"step {t}: {k} of another slot than {c} changed"
        return c

    def unchanged(self, when):
        """The rollout is exactly as after the last check"""
        now = snapshot(self.roll)
        for k in now:
            assert np.array_equal(now[k], self.prev[k]), f"{when}: the rollout's {k} changed"


def run_rollout_lockstep(ctrl, dut, steps, slots, plan=None, before=None, after=None, action_seed=0, blob_every=4, roll=None):
    """ctrl (a handle without the rollout) and dut (the rollout requested here, or `roll` if given) stepped together with
    mt19937 actions; plan(t, actions) may change them in place, before(t, actions) runs ahead of the step and after(t)
    behind it. Every step: equal outputs, the rollout's invariant, equal state blobs every `blob_every` steps. At the
    end: every blob and error bit equal. Returns the RolloutCheck."""
    n = ctrl.num
    roll = roll or RolloutCheck(dut, slots)
    assert_same_observation(ctrl, dut, -1)
    acts = mt19937_actions(action_seed, n, steps)
    for t in range(steps):
        a = acts[t].copy()
        if plan:
            plan(t, a)
        if before:
            before(t, a)
        ctrl.act(a)
        dut.act(a)
        assert_same_observation(ctrl, dut, t)
        rew, ob, first = dut.observe()
        roll.check(t, rew, ob["rgb"], first)
        if after:
            after(t)
        if t % blob_every == 0:
            for e in range(n):
                assert ctrl.get_state(e) == dut.get_state(e), f"step {t} env {e}: state blobs differ"
    for e in range(n):
        assert ctrl.get_state(e) == dut.get_state(e), f"env {e}: state blobs differ at the end"
    er, ed = error_bits(ctrl), error_bits(dut)
    assert np.array_equal(er, ed), f"error bits differ at envs {np.nonzero(er != ed)[0][:8]}"
    return roll
