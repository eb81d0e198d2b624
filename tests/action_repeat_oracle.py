"""Test helpers for action repeat (pgb200_get_action_repeat).

The reference has no action repeat, but it plays one exactly: a step with repeat counts r is a run of plain steps of
the oracle, one per game step. After each, the envs that were not to play it (paused, their level already ended in
this step, or their count used up) are set back to their state before it by set_state, which also re-runs
Game::observe on it (as pause_oracle.py does for a paused env). The rewards of the envs that played are summed in
float32. A level ends where first is set, or where a completed level of use_sequential_levels goes on (first = 0 and
prev_level_complete = 1)."""
import ctypes as C

import numpy as np

from helpers import lib_array, read_lib_array, write_lib_array
from level_seed_oracle import emulate_step, next_level_seeds
from oracle.ref_env import mt19937_actions
from pause_oracle import pause_mask


def action_repeat(env):
    """The int32 repeat counts of a libenv-ABI env of the library under test (oracle.ref_env.RefVecEnv), as
    helpers.lib_array."""
    lib = env.lib
    lib.pgb200_get_action_repeat.argtypes = [C.c_void_p, C.POINTER(C.POINTER(C.c_int32))]
    lib.pgb200_get_action_repeat.restype = C.c_int
    ptr = C.POINTER(C.c_int32)()
    assert lib.pgb200_get_action_repeat(C.c_void_p(env.h), C.byref(ptr)) == 0
    return lib_array(env, ptr, (env.num,), "<i4")


def level_ended(ref):
    """Where the level of `ref`'s envs ended in its last step"""
    return (ref.first != 0) | (ref.info["prev_level_complete"] != 0)


def emulate_repeat_step(ref, actions, reps, paused=None, overrides=None, final=None):
    """One step of `ref` (any libenv-ABI env) as the library takes it with repeat counts `reps`, the pause mask
    `paused` (bool [n] or None) and, if given, the override array holding `overrides` (-1 = none). final: the oracle's
    final outputs (final_obs_oracle.OracleFinal), prepared before each game step. Returns (rew: the float32 sums, the
    game steps each env played, the envs whose reset took their override, level_end, the final frames). The caller then
    observes `ref`: its rew is to be replaced by the sums, and rew and first are 0 on the paused envs."""
    n = ref.num
    count = np.maximum(np.asarray(reps, np.int64), 1)
    live = np.ones(n, bool) if paused is None else ~np.asarray(paused, bool)
    ov = None if overrides is None else np.asarray(overrides, np.int64).copy()
    rew = np.zeros(n, np.float32)
    played = np.zeros(n, np.int64)
    level_end = np.zeros(n, np.uint8)
    frames = np.zeros((n, 64, 64, 3), np.uint8)
    took_all = []
    while live.any():
        still = np.nonzero(~live)[0]
        pre = {int(e): ref.get_state(int(e)) for e in still}
        if final is not None:
            final.prepare(actions)
            level_end[live] = final.level_end[live]
            frames[live] = final.rgb[live]
        if ov is not None:
            _, took = emulate_step(ref, actions, np.where(live, ov, -1))
            ov[took] = -1
            took_all += took
        else:
            ref.act(actions)
        for e, blob in pre.items():
            ref.set_state(e, blob)
        r, _, _ = ref.observe()
        rew[live] += r[live]
        played[live] += 1
        live &= ~level_ended(ref) & (played < count)
    return rew, played, sorted(took_all), level_end, frames


# ---- repeat counts: plan(t) -> int32 [n]
def mixed_plan(n, seed, choices=(-2, 0, 1, 1, 2, 3, 4, 7)):
    """Every step a fresh random count per env, including 0 and negative counts (one game step each)"""
    def plan(t):
        return np.random.RandomState([seed, t]).choice(np.asarray(choices, np.int32), size=n)

    return plan


def constant_plan(n, r):
    def plan(t):
        return np.full(n, r, np.int32)

    return plan


def run_repeat_lockstep(ref, dut, steps, repeat_plan, pause_plan=None, plan=None, overrides=False, final=None,
                        action_seed=0, blob_every=1, before=None):
    """ref (the oracle) and dut (the library under test, its repeat counts requested here) stepped together with
    mt19937 actions. Before step t, repeat_plan(t) gives the counts, pause_plan(t, first) (if given) the paused set,
    and plan(t, actions, pending) may change the step's actions in place and returns {env: seed} to write into dut's
    override array (overrides=True). Every step: dut's outputs equal the emulation's, the state blobs before the step
    are equal every `blob_every` steps, final outputs (final: final_obs_oracle.OracleFinal) are equal where a level
    ended and unchanged elsewhere, and neither the counts nor the override array hold anything but what the step
    defines. before(t), if given, runs first in step t. Returns the game steps played, [steps, n]."""
    from final_obs_oracle import LibFinal

    n = ref.num
    rep = action_repeat(dut)
    assert (read_lib_array(rep) == 1).all(), "new repeat counts are 1 everywhere"
    mask = pause_mask(dut) if pause_plan is not None else None
    seeds = next_level_seeds(dut) if overrides else None
    dut_fin = LibFinal(dut) if final is not None else None
    pending = np.full(n, -1, np.int64)
    acts = mt19937_actions(action_seed, n, steps)
    first = np.zeros(n, np.uint8)
    if dut_fin is not None:
        _, dut_rgb = dut_fin.read()
    hist = np.zeros((steps, n), np.int64)
    for t in range(steps):
        if before:
            before(t)
        a = acts[t].copy()
        r = np.asarray(repeat_plan(t), np.int32)
        paused = np.asarray(pause_plan(t, first), bool) if pause_plan is not None else np.zeros(n, bool)
        new = plan(t, a, pending.copy()) if plan else {}
        write_lib_array(rep, r)
        if mask is not None:
            write_lib_array(mask, paused)
        if overrides:
            for e, s in new.items():
                pending[e] = s
            write_lib_array(seeds, pending)
        if t % blob_every == 0:
            for e in range(n):
                assert dut.get_state(e) == ref.get_state(e), f"step {t} env {e}: state blobs before the step differ"
        rew, played, took, le_r, rgb_r = emulate_repeat_step(ref, a, r, paused, pending if overrides else None, final)
        dut.act(a)
        _, o1, f1 = ref.observe()
        f1 = np.where(paused, 0, f1)
        r2, o2, f2 = dut.observe()
        assert np.array_equal(rew, r2), f"step {t}: rew differs at envs {np.nonzero(rew != r2)[0][:8]}"
        assert np.array_equal(f1, f2), f"step {t}: first differs at envs {np.nonzero(f1 != f2)[0][:8]}"
        for k in ref.info:
            bad = np.nonzero(ref.info[k] != dut.info[k])[0]
            assert len(bad) == 0, f"step {t}: info[{k}] differs at envs {bad[:8]}"
        if not np.array_equal(o1["rgb"], o2["rgb"]):
            bad = np.nonzero((o1["rgb"] != o2["rgb"]).reshape(n, -1).any(1))[0]
            raise AssertionError(f"step {t}: rgb differs at envs {bad[:8]} (counts {r[bad[:8]]}, played {played[bad[:8]]})")
        if final is not None:
            ended = le_r != 0
            le_d, rgb_d = dut_fin.read()
            assert np.array_equal(le_r, le_d), f"step {t}: level_end differs at envs {np.nonzero(le_r != le_d)[0][:8]}"
            assert np.array_equal(rgb_r[ended], rgb_d[ended]), f"step {t}: final frames differ"
            assert np.array_equal(rgb_d[~ended], dut_rgb[~ended]), f"step {t}: a final frame changed where no level ended"
            dut_rgb = rgb_d
        if overrides:
            pending[took] = -1
            assert np.array_equal(read_lib_array(seeds), pending), f"step {t}: override array"
        assert np.array_equal(read_lib_array(rep), r), f"step {t}: the step changed the repeat counts"
        first = f2.copy()
        hist[t] = played
    for e in range(n):
        assert ref.get_state(e) == dut.get_state(e), f"env {e}: state blobs differ at the end"
    if hasattr(dut.lib, "pgb200_get_errors"):
        dut.lib.pgb200_get_errors.restype = C.c_uint32
        assert dut.lib.pgb200_get_errors(C.c_void_p(dut.h), None) == 0
    return hist
