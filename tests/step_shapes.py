"""The step-shape matrix: one lockstep driver for any combination of the six opt-ins of a step, against the oracle.

A step's kernels come from its shape (StepShape, pg_launch.cuh): level choice, pause mask, final outputs, level bank,
level lookahead and rollout. The oracle's outputs depend only on the first three, the semantic shape; a bank, lookahead
and a rollout change nothing but speed. run_shape_lockstep() therefore calls the oracle (observe, get_state, set_state,
act) in a sequence that depends only on the case and the semantic shape, so that the 8 variants of one semantic shape
replay one record (record_key), and checks the library under test against it every step: outputs, final outputs,
override array, pause mask, rollout, state blobs and kernel launches. Records: STEP_SHAPE_RECORDS."""
import ctypes as C
import itertools
import os
import struct

import numpy as np

from final_obs_oracle import LibFinal, final_oracle_env
from helpers import read_lib_array, write_lib_array
from level_bank import build_bank, error_bits
from level_lookahead import enable_lookahead, lookahead_info, resets
from level_seed_oracle import field_offsets, next_level_seeds, patch_fields
from oracle.record import STANDIN_PACK, oracle_env, use_records
from oracle.ref_env import RefVecEnv, mt19937_actions
from oracle.state_blob import parse
from pause_oracle import assert_same_paused_observation, emulate_pause_step, halves_plan, pause_mask
from rollout import RolloutCheck

STEP_SHAPE_RECORDS = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "step_shape_records.json.gz")

OPT_INS = ("level_choice", "pause", "final", "bank", "look", "roll")
SEMANTIC = ("level_choice", "pause", "final")   # the opt-ins the outputs depend on
SHAPES = [dict(zip(OPT_INS, bits)) for bits in itertools.product((False, True), repeat=len(OPT_INS))]
ALL_ON = dict.fromkeys(OPT_INS, True)
ALL16 = "bigfish,bossfight,caveflyer,chaser,climber,coinrun,dodgeball,fruitbot,heist,jumper,leaper,maze,miner,ninja,plunder,starpilot"

# The inputs of every case: num_levels = 0, so that lookahead's predictions hit; a bank of seeds 0..199 and overrides
# drawn from [0, 400), so that some overrides hit the bank and some miss it; a rollout of 5 slots, which the run wraps
# 6 times. Before the checked steps, PRELUDE plain steps on both handles take the agents into their levels, so that the
# games end levels by themselves within the run. Then the envs have three roles, by env % 4: 0 sets action -1 about two
# steps in 3 (one action in 6 in all); 1 starts STEPS_LEFT steps from its time limit, so that the pause windows cross
# it; 2 and 3 play on until their games end their levels.
STEPS = 32
PRELUDE = 100
SLOTS = 5
BANK_SEEDS = range(200)
OVERRIDE_SEEDS = (0, 400)
STEPS_LEFT = 10
BLOB_EVERY = 4
# case: (env name, distribution mode, envs, launch shape of the library under test, extra options)
CASES = {
    "one_game": ("coinrun", "easy", 32, None, {}),
    # 16 games x 5 chunks = 80 launches a step, more than the 64 ticket slots; chunks of 1 and 2 envs
    "sixteen_games": (ALL16, "hard", 96, (5, False), {}),
    # the whole-world view (center_agent=False) of two games, 3 uneven chunks each
    "whole_world": ("caveflyer,jumper", "hard", 32, (3, False), {"center_agent": False}),
}


def shape_id(shape):
    return "+".join(k for k in OPT_INS if shape[k]) or "plain"


def semantic_id(shape):
    return "+".join(k for k in SEMANTIC if shape[k]) or "plain"


def record_key(case, label):
    """The record a run of `case` replays: label is the semantic shape, or the name of a mid-run order"""
    return f"step_shapes::{case}[{label}]#0"


def use_step_shape_records():
    use_records(STEP_SHAPE_RECORDS)


def case_shapes(case):
    """(shape, launch shape) of every run of the GPU matrix for `case`. The 16-game list runs all 64 shapes; one game
    runs its 8 semantic shapes with bank, lookahead and rollout all off and all on (the host debug build runs all 64)."""
    ls = CASES[case][3]
    if case == "one_game":
        return [(s, ls) for s in semantic_shapes(False) + semantic_shapes(True)]
    if case == "sixteen_games":
        return [(s, ls) for s in SHAPES] + [(ALL_ON, (5, True))]
    # whole_world: every render instantiation of the view, behind finish kernels that take overrides from the bank,
    # the slots and generation
    return [(dict(ALL_ON, pause=p, final=f, roll=r), ls) for p, f, r in itertools.product((False, True), repeat=3)]


def semantic_shapes(transparent=True):
    """The 8 semantic shapes, with bank, lookahead and rollout all on (or all off)"""
    return [dict(zip(OPT_INS, bits + (transparent,) * 3)) for bits in itertools.product((False, True), repeat=3)]


def expected_launches(shape, launches_per_step):
    """Kernel launches of one step. Per (game, env chunk) launch, a plain step issues 3: logic, setup and render. A
    two-phase step without final outputs (a level bank or level lookahead) issues 4, with the finish kernel. A step with
    final outputs issues 6: it renders in both phases. Level lookahead adds its own kernel. The rollout adds one per
    step, the advance of its cursor. The level-seed overrides and the pause mask select other instantiations of the same
    kernels and add none."""
    if shape["final"]:
        per_launch = 6
    elif shape["bank"] or shape["look"]:
        per_launch = 4
    else:
        per_launch = 3
    if shape["look"]:
        per_launch += 1
    return per_launch * launches_per_step + (1 if shape["roll"] else 0)


def launches_per_step(name, launch_shape):
    return len(name.split(",")) * (launch_shape[0] if launch_shape else 1)


def kernel_launches(env):
    env.lib.pgb200_kernel_launches.argtypes = [C.c_void_p]
    env.lib.pgb200_kernel_launches.restype = C.c_int64
    return env.lib.pgb200_kernel_launches(C.c_void_p(env.h))


def make_handles(case, lib_path, label, final, launch_shape=None):
    """(the oracle_env replaying record_key(case, label), its final outputs or None, the library under test)"""
    name, mode, n, _, extra = CASES[case]
    kw = dict(distribution_mode=mode, num_levels=0, start_level=0, rand_seed=0, **extra)
    if final:
        ref, ref_fin = final_oracle_env(n, name, lib_path, key=record_key(case, label), **kw)
    else:
        ref, ref_fin = oracle_env(n, name, lib_path, key=record_key(case, label), **kw), None
    dut = RefVecEnv(n, name, lib_path=lib_path, resource_root=STANDIN_PACK, launch_shape=launch_shape, **kw)
    return ref, ref_fin, dut


def request(env, shape, have=None):
    """Turn on the opt-ins of `shape` on env (a libenv-ABI handle of the library under test) that `have` (what an
    earlier call returned) does not hold yet, and only those: requesting the pause mask or the override array selects
    their instantiations even while they hold nothing. Returns {"seeds", "mask", "final", "roll"} as far as requested."""
    have = {} if have is None else have
    if shape["level_choice"] and "seeds" not in have:
        have["seeds"] = next_level_seeds(env)
        assert (read_lib_array(have["seeds"]) == -1).all()
    if shape["pause"] and "mask" not in have:
        have["mask"] = pause_mask(env)
        assert not read_lib_array(have["mask"]).any()
    if shape["final"] and "final" not in have:
        have["final"] = LibFinal(env)
    if shape["bank"] and "bank" not in have:
        assert build_bank(env, BANK_SEEDS) == 0
        have["bank"] = True
    if shape["look"] and "look" not in have:
        assert enable_lookahead(env) == 0
        have["look"] = True
    if shape["roll"] and "roll" not in have:
        have["roll"] = RolloutCheck(env, SLOTS)
    return have


# the actions lean right (7 RIGHT, 8 RIGHT+UP, 6 RIGHT+DOWN): the platformers' agents move on into their levels
LEAN_RIGHT = np.array([7, 8, 7, 8, 6, 5, 7, 8, 2, 4, 10, 11, 12, 13, 14], np.int32)


def _plan(n, t, actions, seed=2):
    """Step t's actions, forced resets and override refills, in place on `actions`: mt19937 actions leaning right; the
    envs of role 0 (env % 4 == 0) set action -1 with p = 2/3 (about one action in 6 in all), the others never. Returns (a seed drawn from OVERRIDE_SEEDS per env, whether an empty entry of env is refilled: p = 1/2,
    so that some resets take no override and are served from their lookahead slots)."""
    rs = np.random.RandomState([seed, t])
    actions[:] = LEAN_RIGHT[actions]
    actions[(rs.randint(3, size=n) < 2) & (np.arange(n) % 4 == 0)] = -1
    return rs.randint(*OVERRIDE_SEEDS, size=n).astype(np.int64), rs.randint(2, size=n) == 1


def _prelude(ref, dut):
    """PRELUDE plain steps of both handles, unchecked, then the envs of role 1 STEPS_LEFT steps from their time limit:
    cur_time patched into their state blobs (the games' limits differ)."""
    n = ref.num
    for a in mt19937_actions(7, n, PRELUDE):
        ref.act(LEAN_RIGHT[a])
        dut.act(LEAN_RIGHT[a])
    for e in range(1, n, 4):
        blob = ref.get_state(e)
        blob = patch_fields(blob, cur_time=parse(blob)["timeout"] - STEPS_LEFT)
        ref.set_state(e, blob)
        dut.set_state(e, blob)


def _timed_out(blob):
    """The step that starts from `blob` reaches the time limit (Game::step: cur_time + 1 >= timeout)"""
    offs = field_offsets(blob)
    cur, timeout = (struct.unpack_from("<i", blob, offs[k][0])[0] for k in ("cur_time", "timeout"))
    return cur + 1 >= timeout


def run_shape_lockstep(case, shape, ref, ref_fin, dut, launch_shape=None, turn_on=None, steps=STEPS):
    """ref (an oracle_env), ref_fin (its final outputs, final_obs_oracle.final_oracle_env; None without final) and dut
    (the library under test, nothing requested, made with `launch_shape`: by default the case's) of `case`, stepped
    together for `steps` steps. The opt-ins of `shape`
    are requested on dut before the first observation, or, with turn_on = {opt-in: step}, right before that step.

    First the prelude (_prelude). Then every step: the paused set P is a random half of the envs while the pause mask is
    on, and the envs of role 0 force about two actions in 3 to -1 (on P too, where the step ignores it). Half the empty override entries are refilled from
    OVERRIDE_SEEDS.
    rew, rgb, first and every info equal the emulation's (rew and first 0 on P); level_end and the final frames equal
    the oracle's (level_end 0 on P, final frames unchanged where no level ended); the overrides taken read -1 and were
    played, every other entry keeps its value, and no env in P takes its entry; the mask is unchanged; the rollout
    holds the step's outputs; the kernel launches are expected_launches(); the state blobs before the step are equal
    every BLOB_EVERY steps. At the end: every state blob, error bits 0, and the lookahead counters account for every
    reset. Returns counts of what the run covered (assert_coverage)."""
    name = CASES[case][0]
    lps = launches_per_step(name, launch_shape or CASES[case][3])
    n = ref.num
    turn_on = turn_on or {}
    _prelude(ref, dut)
    on = {k: shape[k] and turn_on.get(k, 0) <= 0 for k in OPT_INS}
    have = request(dut, on)
    acts = mt19937_actions(0, n, steps)
    halves = halves_plan(n, 1)
    pending = np.full(n, -1, np.int64)
    stats = dict(game=0, timeout=0, caller=0, taken=0, held=0, resets=0)
    look_from = 0
    assert_same_paused_observation(ref, dut, np.zeros(n, bool), -1)
    fin_rgb = have["final"].read()[1] if "final" in have else None
    for t in range(steps):
        was = on
        on = {k: shape[k] and turn_on.get(k, 0) <= t for k in OPT_INS}
        if on != was:
            have = request(dut, on, have)
            if on["final"] and not was["final"]:
                fin_rgb = have["final"].read()[1]
            if on["look"] and not was["look"]:
                look_from = t
        a = acts[t].copy()
        fresh, refill = _plan(n, t, a)
        paused = halves(t, None) if on["pause"] else np.zeros(n, bool)
        if on["level_choice"]:
            pending = np.where((pending < 0) & refill, fresh, pending)
            write_lib_array(have["seeds"], pending)
            stats["held"] += int((paused & (a == -1) & (pending >= 0)).sum())
        if on["pause"]:
            write_lib_array(have["mask"], paused)
        if on["final"]:
            ref_fin.prepare(a)
        pre, took = emulate_pause_step(ref, a, paused, pending if on["level_choice"] else None)
        if t % BLOB_EVERY == 0:
            for e in range(n):
                assert dut.get_state(e) == pre[e], f"step {t} env {e}: state blobs before the step differ"
        before = kernel_launches(dut)
        dut.act(a)
        got = kernel_launches(dut) - before
        assert got == expected_launches(on, lps), f"step {t}: {got} kernel launches, {shape_id(on)} issues {expected_launches(on, lps)}"
        assert_same_paused_observation(ref, dut, paused, t)
        rew, ob, first = dut.rew, dut.rgb, dut.first.astype(bool)
        if on["final"]:
            le_r, rgb_r = ref_fin.read()
            le_r[paused] = 0
            ended = le_r != 0
            ref._fold(le_r, rgb_r[ended])
            le_d, rgb_d = have["final"].read()
            assert np.array_equal(le_r, le_d), f"step {t}: level_end differs at envs {np.nonzero(le_r != le_d)[0][:8]}"
            if not np.array_equal(rgb_r[ended], rgb_d[ended]):
                bad = np.nonzero(ended & (rgb_r != rgb_d).reshape(n, -1).any(1))[0]
                raise AssertionError(f"step {t}: final frames differ at envs {bad[:8]}")
            assert np.array_equal(rgb_d[~ended], fin_rgb[~ended]), f"step {t}: a final frame changed where no level ended"
            assert np.array_equal(ended, first), f"step {t}: level_end set at envs {np.nonzero(ended != first)[0][:8]} against first"
            fin_rgb = rgb_d
        if on["level_choice"]:
            # the emulation never lets a paused env take its entry; a paused env of dut that took one fails the array check
            assert np.array_equal(dut.info["level_seed"][took], pending[took]), f"step {t}: an override taken was not played"
            pending[took] = -1
            now = read_lib_array(have["seeds"])
            assert np.array_equal(now, pending), f"step {t}: override array differs at envs {np.nonzero(now != pending)[0][:8]}"
            stats["taken"] += len(took)
        if on["pause"]:
            assert np.array_equal(read_lib_array(have["mask"]), paused.astype(np.uint8)), f"step {t}: the step changed the mask"
        if on["roll"]:
            have["roll"].check(t, rew, ob, dut.first)
        assert not (first & paused).any()
        for e in np.nonzero(first)[0]:
            cause = "caller" if a[e] == -1 else "timeout" if _timed_out(pre[e]) else "game"
            stats[cause] += 1
        if on["look"]:
            stats["resets"] += int(first.sum())
    for e in range(n):
        assert ref.get_state(e) == dut.get_state(e), f"env {e}: state blobs differ at the end"
    err = error_bits(dut)
    assert not err.any(), f"error bits {err[err != 0][:8]} at envs {np.nonzero(err)[0][:8]}"
    if shape["look"]:
        info = lookahead_info(dut)
        stats.update((k, info[k]) for k in ("served", "bank", "generated"))
        assert resets(info) == stats["resets"], f"{stats['resets']} resets since step {look_from}, lookahead counters {info}"
    return stats


def assert_coverage(shape, stats):
    """The run ended levels in all three ways, took overrides and held some in paused envs, and (bank + lookahead +
    level choice) served resets from the slots and the bank and generated others."""
    for cause in ("game", "timeout", "caller"):
        assert stats[cause] > 0, f"no level ended by {cause}: {stats}"
    if shape["level_choice"]:
        assert stats["taken"] > 0, f"no override taken: {stats}"
        if shape["pause"]:
            assert stats["held"] > 0, f"no paused env held an override: {stats}"
    if shape["look"]:
        assert stats["served"] > 0, f"no reset served from a lookahead slot: {stats}"
        if shape["level_choice"]:
            assert stats["generated"] > 0, f"no override generated: {stats}"
            if shape["bank"]:
                assert stats["bank"] > 0, f"no override served from the bank: {stats}"


def run_case(case, lib_path, shape, launch_shape=None, turn_on=None, label=None):
    """One run of the matrix: handles made, run_shape_lockstep, coverage asserted, handles closed. Returns the counts."""
    launch_shape = launch_shape or CASES[case][3]
    ref, ref_fin, dut = make_handles(case, lib_path, label or semantic_id(shape), shape["final"], launch_shape)
    stats = run_shape_lockstep(case, shape, ref, ref_fin, dut, launch_shape=launch_shape, turn_on=turn_on)
    assert_coverage(shape, stats)
    for env in (ref, ref_fin, dut):
        if env is not None:
            env.close()
    return stats


# Opt-ins turned on mid-run, one every 4 steps from step 4, in three orders; each order has its own record
MID_RUN_ORDERS = {
    "forward": OPT_INS,
    "reverse": OPT_INS[::-1],
    "shuffled": ("look", "final", "roll", "level_choice", "bank", "pause"),
}


def mid_run_turn_on(order):
    return {k: 4 * (i + 1) for i, k in enumerate(MID_RUN_ORDERS[order])}
