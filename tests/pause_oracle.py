"""Test helpers for the per-env pause mask (pgb200_get_pause_mask).

The reference has no pause, but its wire format expresses one exactly: a paused env's step is a plain step
followed by set_state of the env's pre-step blob, which restores every byte of its state and re-runs
Game::observe on it (its rgb and infos). emulate_pause_step() builds a step with paused set P that way on any
implementation of the libenv ABI (the oracle itself, or the oracle's records replayed through the library under
test). The library's outputs are then the emulation's, except that rew and first are 0 on P. Combined with level
choice, an env in P does not take its override; combined with final outputs, level_end is 0 on P.

The pause patterns are deterministic functions of (seed, step, env), or of the outputs of the previous step.
Records: PAUSE_RECORDS, apart from tests/golden/oracle_records.json.gz.
"""
import ctypes as C
import os

import numpy as np

from helpers import lib_array, read_lib_array, write_lib_array
from level_seed_oracle import emulate_step, next_level_seeds
from oracle.ref_env import mt19937_actions

PAUSE_RECORDS = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "pause_records.json.gz")


def use_pause_records():
    """Make the records of PAUSE_RECORDS replayable through oracle.record.oracle_env."""
    from oracle.record import use_records

    use_records(PAUSE_RECORDS)


def pause_mask(env):
    """The uint8 pause mask of a libenv-ABI env of the library under test (oracle.ref_env.RefVecEnv), as
    helpers.lib_array."""
    lib = env.lib
    lib.pgb200_get_pause_mask.argtypes = [C.c_void_p, C.POINTER(C.POINTER(C.c_uint8))]
    lib.pgb200_get_pause_mask.restype = C.c_int
    ptr = C.POINTER(C.c_uint8)()
    assert lib.pgb200_get_pause_mask(C.c_void_p(env.h), C.byref(ptr)) == 0
    return lib_array(env, ptr, (env.num,), "|u1")


def emulate_pause_step(ref, actions, paused, overrides=None):
    """One step of `ref` (any libenv-ABI env) as the library takes it with the pause mask `paused` (bool [n]) and,
    if given, the override array holding `overrides` (-1 = none). Returns (the pre-step state blobs of every env,
    the envs whose reset took their override). The caller then observes `ref` and sets rew and first to 0 on the
    paused envs."""
    n = ref.num
    if overrides is not None:
        ov = np.where(paused, -1, overrides)
        pre, took = emulate_step(ref, actions, ov)
    else:
        pre = [ref.get_state(e) for e in range(n)]
        ref.act(actions)
        took = []
    for e in np.nonzero(paused)[0]:
        ref.set_state(int(e), pre[e])
    return pre, took


def observe_paused(ref, paused):
    """ref.observe() with rew and first set to 0 on the paused envs: the library's outputs of a paused step."""
    r, o, f = ref.observe()
    r, f = r.copy(), f.copy()
    r[paused] = 0
    f[paused] = 0
    return r, o, f


def assert_same_paused_observation(ref, dut, paused, t):
    r1, o1, f1 = observe_paused(ref, paused)
    r2, o2, f2 = dut.observe()
    assert np.array_equal(r1, r2), f"step {t}: rew differs at envs {np.nonzero(r1 != r2)[0][:8]}"
    assert np.array_equal(f1, f2), f"step {t}: first differs at envs {np.nonzero(f1 != f2)[0][:8]}"
    for k in ref.info:
        bad = np.nonzero(ref.info[k] != dut.info[k])[0]
        assert len(bad) == 0, f"step {t}: info[{k}] differs at envs {bad[:8]}"
    if not np.array_equal(o1["rgb"], o2["rgb"]):
        bad = np.nonzero((o1["rgb"] != o2["rgb"]).reshape(ref.num, -1).any(1))[0]
        raise AssertionError(f"step {t}: rgb differs at envs {bad[:8]} (paused: {paused[bad[:8]]})")


# ---- pause patterns: plan(t, first) -> bool [n], first = the outputs' first of the previous step
def halves_plan(n, seed):
    """Every step a fresh random half of the envs is paused."""
    def plan(t, first):
        return np.random.RandomState([seed, t]).randint(2, size=n).astype(bool)

    return plan


def long_plan(n, seed, start=(0, 8), length=(20, 60)):
    """Env e is paused for one window [a_e, a_e + L_e) of steps: with the time limit 10 steps ahead, the windows span
    the step at which the env would have timed out."""
    rs = np.random.RandomState(seed)
    a = rs.randint(*start, size=n)
    L = rs.randint(*length, size=n)

    def plan(t, first):
        return (t >= a) & (t < a + L)

    return plan


def episode_end_plan(n, release_every=None):
    """The evaluation pattern: an env is paused from the step after its level ended (first set), and stays paused.
    With release_every, all envs are released every release_every steps (aligned episodes)."""
    state = {"paused": np.zeros(n, bool)}

    def plan(t, first):
        if release_every and t % release_every == 0:
            state["paused"][:] = False
        else:
            state["paused"] |= first.astype(bool)
        return state["paused"].copy()

    return plan


def all_plan(n, window=(10, 40)):
    """Every env paused in a window of steps."""
    def plan(t, first):
        return np.full(n, window[0] <= t < window[1])

    return plan


def zero_plan(n):
    def plan(t, first):
        return np.zeros(n, bool)

    return plan


def run_pause_lockstep(ref, dut, steps, pause_plan, plan=None, overrides=False, final=None, action_seed=0,
                       blob_every=1, before=None, force_paused=False):
    """ref (the oracle, or an oracle_env) and dut (the library under test, its pause mask requested here) stepped
    together with mt19937 actions. Before step t, pause_plan(t, first) gives the paused set P, plan(t, actions,
    pending) may change the step's actions in place and returns {env: seed} to write into dut's override array
    (overrides=True), and force_paused=True sets the actions of P to -1. Every step: dut's outputs equal the
    emulation's (rew and first 0 on P), state blobs before the step are equal every `blob_every` steps, and the
    override entries of P are neither read nor consumed. final = (the oracle's final outputs, as
    final_obs_oracle.final_oracle_env returns them): level_end equal with 0 on P, final frames equal where a level
    ended and unchanged elsewhere. before(t), if given, runs first in step t. Returns the paused sets, [steps, n]."""
    from final_obs_oracle import LibFinal

    n = ref.num
    mask = pause_mask(dut)
    assert not read_lib_array(mask).any(), "a new pause mask holds 0 everywhere"
    seeds = next_level_seeds(dut) if overrides else None
    dut_fin = LibFinal(dut) if final is not None else None
    checked = hasattr(ref, "_fold")
    pending = np.full(n, -1, np.int64)
    acts = mt19937_actions(action_seed, n, steps)
    first = np.zeros(n, np.uint8)
    assert_same_paused_observation(ref, dut, np.zeros(n, bool), -1)
    if dut_fin is not None:
        _, dut_rgb = dut_fin.read()
    hist = np.zeros((steps, n), bool)
    for t in range(steps):
        if before:
            before(t)
        a = acts[t].copy()
        paused = np.asarray(pause_plan(t, first), bool)
        new = plan(t, a, pending.copy()) if plan else {}
        if force_paused:
            a[paused] = -1
        write_lib_array(mask, paused)
        if overrides:
            for e, s in new.items():
                pending[e] = s
            write_lib_array(seeds, pending)
        if final is not None:
            final.prepare(a)
        pre, took = emulate_pause_step(ref, a, paused, pending if overrides else None)
        if t % blob_every == 0:
            for e in range(n):
                assert dut.get_state(e) == pre[e], f"step {t} env {e}: state blobs before the step differ"
        dut.act(a)
        assert_same_paused_observation(ref, dut, paused, t)
        first = dut.first.copy()
        if final is not None:
            le_r, rgb_r = final.read()
            le_r[paused] = 0
            ended = le_r != 0
            if checked:
                ref._fold(le_r, rgb_r[ended])
            le_d, rgb_d = dut_fin.read()
            assert np.array_equal(le_r, le_d), f"step {t}: level_end differs at envs {np.nonzero(le_r != le_d)[0][:8]}"
            assert np.array_equal(rgb_r[ended], rgb_d[ended]), f"step {t}: final frames differ"
            assert np.array_equal(rgb_d[~ended], dut_rgb[~ended]), f"step {t}: a final frame changed where no level ended"
            dut_rgb = rgb_d
        if overrides:
            assert not paused[took].any()
            pending[took] = -1
            assert np.array_equal(read_lib_array(seeds), pending), f"step {t}: override array"
        assert np.array_equal(read_lib_array(mask), paused.astype(np.uint8)), f"step {t}: the step changed the mask"
        hist[t] = paused
    for e in range(n):
        assert ref.get_state(e) == dut.get_state(e), f"env {e}: state blobs differ at the end"
    if hasattr(dut.lib, "pgb200_get_errors"):
        dut.lib.pgb200_get_errors.restype = C.c_uint32
        assert dut.lib.pgb200_get_errors(C.c_void_p(dut.h), None) == 0
    return hist


def check_set_state_into_paused_env(ref, dut, steps=30):
    """set_state into a paused env loads the state, re-renders it, and the env stays paused: the next steps leave
    it as loaded. ref and dut: same game, same env count; ref is only a donor of states."""
    n = dut.num
    mask = pause_mask(dut)
    paused = np.zeros(n, bool)
    paused[::2] = True
    write_lib_array(mask, paused)
    acts = mt19937_actions(3, n, steps)
    for t in range(steps):
        ref.act(acts[t])
    ref.observe()
    donor = [ref.get_state(e) for e in range(n)]
    for e in np.nonzero(paused)[0]:
        dut.set_state(int(e), donor[e])
    assert np.array_equal(read_lib_array(mask), paused.astype(np.uint8)), "set_state changed the mask"
    _, ob, _ = dut.observe()
    r_ob = ref.observe()[1]["rgb"]
    assert np.array_equal(ob["rgb"][paused], r_ob[paused]), "set_state did not render the loaded state"
    seen = ob["rgb"].copy()
    for t in range(steps):
        dut.act(acts[t])
        rew, ob, first = dut.observe()
        assert not rew[paused].any() and not first[paused].any()
        assert np.array_equal(ob["rgb"][paused], seen[paused]), f"step {t}: a paused env's frame changed"
    for e in np.nonzero(paused)[0]:
        assert dut.get_state(int(e)) == donor[e], f"env {e}: a paused env's state changed"
