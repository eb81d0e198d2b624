"""Test helpers for per-env level-seed overrides (pgb200_get_next_level_seeds).

The reference has no override, but its own wire format expresses one exactly: Game::reset (game.cpp:93-118)
skips the draw of the next level seed when episodes_remaining != 0, and then also zeroes reward, done and
level_complete. emulate_step() builds an override step out of plain steps, get_state and set_state on any
implementation of the libenv ABI (the oracle itself, or the oracle's records replayed through the library
under test), so a run with overrides can be compared with the reference bit for bit.
"""
import ctypes as C
import os
import struct

import numpy as np

from helpers import lib_array, read_lib_array, write_lib_array
from oracle.state_blob import Reader, parse

# The oracle's recorded outputs of tests/test_gpu_level_seeds.py, kept apart from tests/golden/oracle_records.json.gz
# (which oracle.record reads) so that the records of the existing tests stay as they are. Recorded like those
# (PG_ORACLE_RECORD_DIR), added with oracle.record.merge(<dir>, out=LEVEL_SEED_RECORDS).
LEVEL_SEED_RECORDS = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "level_seed_records.json.gz")


def use_level_seed_records():
    """Make the records of LEVEL_SEED_RECORDS replayable through oracle.record.oracle_env."""
    from oracle.record import use_records

    use_records(LEVEL_SEED_RECORDS)

# the fixed-size scalar header of the blob, in wire order (oracle/state_blob.py parse)
_OPTION_INTS = ["paint_vel_info", "use_generated_assets", "use_monochrome_assets", "restrict_themes", "use_backgrounds",
                "center_agent", "debug_mode", "distribution_mode", "use_sequential_levels", "use_easy_jump", "plain_assets",
                "physics_mode", "grid_step", "level_seed_low", "level_seed_high", "game_type", "game_n"]
_STEP_INTS = ["done", "level_complete", "action", "timeout", "current_level_seed", "prev_level_seed", "episodes_remaining",
              "episode_done", "last_reward_timer"]
_TAIL_INTS = ["default_action", "fixed_asset_seed", "cur_time", "is_waiting_for_step", "grid_size"]


def field_offsets(blob):
    """{field: (byte offset, 'i' or 'f')} of the int / float fields of the blob's scalar header."""
    r = Reader(blob)
    out = {}

    def take(name, kind):
        out[name] = (r.o, kind)
        getattr(r, kind)()

    r.i()
    r.s()
    for k in _OPTION_INTS:
        take(k, "i")
    for _ in ("level_seed_rand_gen", "rand_gen"):
        r.i()
        r.s()
    take("reward", "f")
    for k in _STEP_INTS:
        take(k, "i")
    take("last_reward", "f")
    for k in _TAIL_INTS:
        take(k, "i")
    return out


def patch_fields(blob, **fields):
    """The blob with the named scalar header fields rewritten (everything else byte for byte as it was)."""
    offs = field_offsets(blob)
    out = bytearray(blob)
    for name, value in fields.items():
        o, kind = offs[name]
        struct.pack_into("<i" if kind == "i" else "<f", out, o, value)
    return bytes(out)


def next_level_seeds(env):
    """The int32 override array of a libenv-ABI env of the library under test (oracle.ref_env.RefVecEnv), as
    helpers.lib_array."""
    lib = env.lib
    lib.pgb200_get_next_level_seeds.argtypes = [C.c_void_p, C.POINTER(C.POINTER(C.c_int32))]
    lib.pgb200_get_next_level_seeds.restype = C.c_int
    ptr = C.POINTER(C.c_int32)()
    assert lib.pgb200_get_next_level_seeds(C.c_void_p(env.h), C.byref(ptr)) == 0
    return lib_array(env, ptr, (env.num,), "<i4")


def emulate_step(ref, actions, overrides):
    """One step of `ref` (any libenv-ABI env; no override support needed) as the library takes it with the
    override array holding `overrides` (-1 = none). Returns (the pre-step state blobs of every env, the envs
    whose reset took their override). The caller then observes `ref`.

    1. get_state of every env; act; observe: the plain step. An env with an override that reset in it
       (cur_time == 0) takes the override.
    2. If any did: every env back to its pre-step state, the envs that take an override with
       current_level_seed = s and episodes_remaining = 1 (Game::reset then keeps s and does not advance
       level_seed_rand_gen); the same actions again; then the step outputs those resets zero (reward, done,
       level_complete, episode_done) and prev_level_seed put back to the plain step's values by set_state,
       which re-runs Game::observe."""
    n = ref.num
    pre = [ref.get_state(e) for e in range(n)]
    ref.act(actions)
    ref.observe()
    plain = {}
    for e in range(n):
        if overrides[e] >= 0:
            st = parse(ref.get_state(e))
            if st["cur_time"] == 0:
                plain[e] = st
    if plain:
        for e in range(n):
            blob = pre[e]
            if e in plain:
                blob = patch_fields(blob, current_level_seed=int(overrides[e]), episodes_remaining=1)
            ref.set_state(e, blob)
        ref.act(actions)
        for e, st in plain.items():
            ref.set_state(e, patch_fields(ref.get_state(e), **{k: st[k] for k in ("reward", "done", "level_complete", "episode_done",
                                                                                    "prev_level_seed")}))
    return pre, sorted(plain)


def run_override_lockstep(ref, dut, steps, plan, action_seed=0):
    """ref (the oracle, or its records) and dut (the library under test) stepped together for `steps` steps with
    mt19937 actions. Before step t, plan(t, actions, pending) may change the step's actions in place and returns
    {env: seed} to write into dut's override array (pending = what the array holds now). Every step: the library's
    state blobs before the step equal the emulation's, its outputs after the step equal the emulation's, the
    entries the step's resets took read -1 and every other entry keeps its value. Returns the overrides taken."""
    from helpers import assert_same_observation
    from oracle.ref_env import mt19937_actions

    n = ref.num
    seeds = next_level_seeds(dut)
    pending = read_lib_array(seeds).astype(np.int64)
    assert (pending == -1).all(), "a new override array holds -1 everywhere"
    acts = mt19937_actions(action_seed, n, steps)
    assert_same_observation(ref, dut, -1)
    taken = 0
    for t in range(steps):
        a = acts[t].copy()
        for e, s in plan(t, a, pending.copy()).items():
            pending[e] = s
        write_lib_array(seeds, pending)
        dut_pre = [dut.get_state(e) for e in range(n)]
        pre, took = emulate_step(ref, a, pending)
        for e in range(n):
            assert dut_pre[e] == pre[e], f"step {t} env {e}: state blobs before the step differ"
        dut.act(a)
        assert_same_observation(ref, dut, t)
        for e in took:
            assert dut.info["level_seed"][e] == pending[e], f"step {t} env {e}: override not played"
        pending[took] = -1
        now = read_lib_array(seeds)
        assert np.array_equal(now, pending), f"step {t}: override array {now[now != pending][:8]} where {pending[now != pending][:8]} was expected"
        taken += len(took)
    for e in range(n):
        assert dut.get_state(e) == ref.get_state(e), f"env {e}: state blobs differ at the end"
    return taken


def refill_plan(n, seed, low=0, high=2 ** 31 - 1, force_every=8):
    """Overrides preloaded for every env and refilled as soon as consumed, seeds drawn from [low, high);
    about one action in `force_every` is -1 (a forced reset)."""
    rs = np.random.RandomState(seed)

    def plan(t, actions, pending):
        force = rs.randint(force_every, size=n) == 0
        actions[force] = -1
        empty = np.nonzero(pending < 0)[0]
        return {int(e): int(s) for e, s in zip(empty, rs.randint(low, high, size=len(empty)))}

    return plan


def check_consumed_kept_and_set_state(lib_path, resource_root=None):
    """Consumed entries read -1, untouched entries keep their value, and set_state neither reads nor changes
    the array: a pending override survives loading a state and is taken by the next reset."""
    from oracle.ref_env import RefVecEnv, default_pack

    kw = dict(distribution_mode="hard", num_levels=200, start_level=0, lib_path=lib_path, resource_root=resource_root or default_pack())
    dut = RefVecEnv(8, "coinrun", rand_seed=0, **kw)
    donor = RefVecEnv(8, "coinrun", rand_seed=7, **kw)
    seeds = next_level_seeds(dut)
    want = np.array([100, 101, 102, 103, 104, 105, 106, -1])
    write_lib_array(seeds, want)
    for e in range(8):
        dut.set_state(e, donor.get_state(e))
    assert np.array_equal(read_lib_array(seeds), want)
    for e in range(8):
        assert dut.get_state(e) == donor.get_state(e), "get_state carries no override"
    acts = np.array([-1, -1, -1, -1, 4, 4, 4, -1], np.int32)
    dut.act(acts)
    dut.observe()
    got = read_lib_array(seeds)
    assert np.array_equal(got[:4], [-1] * 4) and np.array_equal(got[4:], want[4:])
    assert np.array_equal(dut.info["level_seed"][:4], want[:4])
    assert dut.first[7] == 1 and read_lib_array(seeds)[7] == -1
    dut.close()
    donor.close()
