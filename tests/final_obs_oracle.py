"""Test helpers for final outputs (pgb200_get_final_outputs): the frame each env's level ended in, and why.

The reference never renders a final state: Game::step (game.cpp:120-155) resets before it observes. One hook,
tests/native/final_frame_hook.cpp, replays game.cpp:121-142 on one env of a reference handle and renders what
Game::observe would; final_frame_hook() builds it (against the reference's headers, linking oracle/_ref/libenv_ref.so)
into tests/_build/ the first time a test needs it. OracleFinal runs the hook on a scratch oracle handle loaded with the
compared oracle's pre-step states, so that oracle is never mutated.
LibFinal reads the arrays of a handle of the library under test.

Records: FINAL_OBS_RECORDS, apart from tests/golden/oracle_records.json.gz. final_oracle_env() returns an
oracle_env (oracle.record) and the source of its final outputs: the hook while recording, the library's own
arrays on replay. run_final_lockstep folds level_end and the final frames of the envs whose level ended into the
oracle_env's running digest after every step, so both modes check the same outputs.
"""
import ctypes as C
import os

import numpy as np

from helpers import assert_same_observation, lib_array, read_lib_array, write_lib_array
from level_seed_oracle import emulate_step, next_level_seeds
from oracle.record import STANDIN_PACK, oracle_env, recording_dir, use_records
from oracle.ref_env import REF_LIB, RefVecEnv, mt19937_actions

HERE = os.path.dirname(os.path.abspath(__file__))
FINAL_OBS_RECORDS = os.path.join(HERE, "golden", "final_obs_records.json.gz")
HOOK_SRC = os.path.join(HERE, "native", "final_frame_hook.cpp")
HOOK_LIB = os.path.join(HERE, "_build", "libfinal_frame_hook.so")
FRAME = (64, 64, 3)


def final_frame_hook():
    """The hook's library, built if it is missing or older than its source or the oracle library. Building needs the
    reference's headers; without them a prebuilt library is used, and without one the calling test is skipped."""
    import subprocess

    import pytest

    from oracle import build_ref

    if not os.path.exists(HOOK_LIB) or os.path.getmtime(HOOK_LIB) < max(os.path.getmtime(HOOK_SRC), os.path.getmtime(REF_LIB)):
        if not build_ref.reference_available():
            if not os.path.exists(HOOK_LIB):
                pytest.skip("final-frame hook not built and reference tree absent")
        else:
            os.makedirs(os.path.dirname(HOOK_LIB), exist_ok=True)
            tmp = f"{HOOK_LIB}.{os.getpid()}.tmp"
            ref_dir = os.path.dirname(REF_LIB)
            rpath = "$ORIGIN/" + os.path.relpath(ref_dir, os.path.dirname(HOOK_LIB))
            subprocess.check_call(["g++", *build_ref.CXXFLAGS, "-shared", HOOK_SRC, "-o", tmp, "-L" + ref_dir,
                                   "-l:" + os.path.basename(REF_LIB), "-Wl,-rpath," + rpath])
            os.replace(tmp, HOOK_LIB)
    lib = C.CDLL(HOOK_LIB)
    lib.final_frame_hook.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p]
    lib.final_frame_hook.restype = C.c_int
    return lib.final_frame_hook


def use_final_obs_records():
    """Make the records of FINAL_OBS_RECORDS replayable through oracle.record.oracle_env."""
    use_records(FINAL_OBS_RECORDS)


class OracleFinal:
    """The oracle's final outputs. `ref` is a reference handle (RefVecEnv on REF_LIB); `scratch` another one with the
    same env count and game list, on the same asset pack. prepare(actions) must be called before `ref` steps."""

    def __init__(self, ref, scratch):
        self.ref, self.scratch = ref, scratch
        self.hook = final_frame_hook()
        self.level_end = np.zeros(ref.num, np.uint8)
        self.rgb = np.zeros((ref.num,) + FRAME, np.uint8)
        self._frame = np.zeros(FRAME, np.uint8)

    def prepare(self, actions):
        for e in range(self.ref.num):
            self.scratch.set_state(e, self.ref.get_state(e))
        for e in range(self.ref.num):
            cause = self.hook(C.c_void_p(self.scratch.h), e, int(actions[e]), self._frame.ctypes.data)
            self.level_end[e] = cause
            if cause:
                self.rgb[e] = self._frame

    def read(self):
        return self.level_end.copy(), self.rgb.copy()

    def close(self):
        self.scratch.close()


class LibFinal:
    """The final outputs of a handle of the library under test (RefVecEnv): host arrays in the host debug build,
    device arrays read through torch in the GPU build. Requesting them turns them on for every later step."""

    def __init__(self, env):
        from procgen_b200.libenv import FinalOutputs

        lib = env.lib
        lib.pgb200_get_final_outputs.argtypes = [C.c_void_p, C.POINTER(FinalOutputs)]
        lib.pgb200_get_final_outputs.restype = C.c_int
        out = FinalOutputs()
        assert lib.pgb200_get_final_outputs(C.c_void_p(env.h), C.byref(out)) == 0
        self._rgb = lib_array(env, out.rgb, (env.num,) + FRAME, "|u1")
        self._level_end = lib_array(env, out.level_end, (env.num,), "|u1")

    def prepare(self, actions):
        pass

    def read(self):
        return read_lib_array(self._level_end), read_lib_array(self._rgb)

    def close(self):
        pass


def oracle_final(ref, num, env_name, pack, **kw):
    """OracleFinal for a live reference handle `ref` made with RefVecEnv(num, env_name, **kw) on `pack`."""
    kw = {k: v for k, v in kw.items() if k not in ("extra_options", "launch_shape", "ob_layout", "lib_path", "resource_root", "pack_path")}
    return OracleFinal(ref, RefVecEnv(num, env_name, lib_path=REF_LIB, pack_path=pack, **kw))


def final_oracle_env(num, env_name, lib_path, key=None, **kw):
    """(oracle_env, its final outputs): the hook on the oracle while recording, the library's arrays on replay."""
    ref = oracle_env(num, env_name, lib_path, key=key, **kw)
    fin = oracle_final(ref.env, num, env_name, STANDIN_PACK, **kw) if recording_dir() else LibFinal(ref.env)
    return ref, fin


def force_plan(seed, every=16):
    """About one action in `every` set to -1 (a reset by the caller)."""
    rs = np.random.RandomState(seed)

    def plan(t, actions, pending):
        actions[rs.randint(every, size=len(actions)) == 0] = -1
        return {}

    return plan


def run_final_lockstep(ref, ref_fin, dut, steps, plan=None, overrides=False, action_seed=0, blob_every=25, sequential=False, before=None):
    """ref (the oracle, or an oracle_env) and dut (the library under test, final outputs requested here) stepped
    together. Before step t, plan(t, actions, pending) may change the step's actions in place and returns
    {env: seed} to write into dut's override array (overrides=True: the oracle then plays the step through
    emulate_step). Every step: the outputs are equal, level_end is equal everywhere, the final frames are equal
    where a level ended and dut's are unchanged elsewhere, and level_end != 0 exactly where first is set (under
    use_sequential_levels a completed level may also report 1 with first = 0). State blobs are compared every
    `blob_every` steps and at the end. before(t), if given, runs first in step t. Returns level_end of every step,
    [steps, envs]."""
    n = ref.num
    dut_fin = LibFinal(dut)
    checked = hasattr(ref, "_fold")
    seeds = next_level_seeds(dut) if overrides else None
    pending = np.full(n, -1, np.int64)
    acts = mt19937_actions(action_seed, n, steps)
    assert_same_observation(ref, dut, -1)
    _, dut_rgb = dut_fin.read()
    ends = np.zeros((steps, n), np.uint8)
    for t in range(steps):
        if before:
            before(t)
        a = acts[t].copy()
        new = plan(t, a, pending.copy()) if plan else {}
        if overrides:
            for e, s in new.items():
                pending[e] = s
            write_lib_array(seeds, pending)
        if t % blob_every == 0:
            for e in range(n):
                assert ref.get_state(e) == dut.get_state(e), f"step {t} env {e}: state blobs differ"
        ref_fin.prepare(a)
        took = []
        if overrides:
            _, took = emulate_step(ref, a, pending)
        else:
            ref.act(a)
        dut.act(a)
        assert_same_observation(ref, dut, t)
        le_r, rgb_r = ref_fin.read()
        le_d, rgb_d = dut_fin.read()
        ended = le_r != 0
        if checked:
            ref._fold(le_r, rgb_r[ended])
        assert np.array_equal(le_r, le_d), f"step {t}: level_end differs at envs {np.nonzero(le_r != le_d)[0][:8]}"
        if not np.array_equal(rgb_r[ended], rgb_d[ended]):
            bad = np.nonzero(ended & (rgb_r != rgb_d).reshape(n, -1).any(1))[0]
            raise AssertionError(f"step {t}: final frames differ at envs {bad[:8]}")
        assert np.array_equal(rgb_d[~ended], dut_rgb[~ended]), f"step {t}: a final frame changed where no level ended"
        first = dut.first != 0
        ok = ended == first
        if sequential:
            ok |= (le_d == 1) & ~first
        assert ok.all(), f"step {t}: level_end {le_d[~ok][:8]} where first is {dut.first[~ok][:8]} (envs {np.nonzero(~ok)[0][:8]})"
        if overrides:
            pending[took] = -1
            assert np.array_equal(read_lib_array(seeds), pending), f"step {t}: override array"
        dut_rgb = rgb_d
        ends[t] = le_d
    for e in range(n):
        assert ref.get_state(e) == dut.get_state(e), f"env {e}: state blobs differ at the end"
    if hasattr(dut.lib, "pgb200_get_errors"):
        dut.lib.pgb200_get_errors.restype = C.c_uint32
        assert dut.lib.pgb200_get_errors(C.c_void_p(dut.h), None) == 0
    return ends


def near_timeout(envs, n, steps_left=10):
    """Put every env of each of `envs` (the same states in all) `steps_left` steps before its time limit: cur_time
    patched into its state blob (the games' limits differ)."""
    from level_seed_oracle import patch_fields
    from oracle.state_blob import parse

    for e in range(n):
        blob = envs[0].get_state(e)
        blob = patch_fields(blob, cur_time=parse(blob)["timeout"] - steps_left)
        for env in envs:
            env.set_state(e, blob)
