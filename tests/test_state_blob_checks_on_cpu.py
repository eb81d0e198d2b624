"""set_state's checks and its readings of the wire format, in the host debug build.

The parity suites compare the blobs the library and the oracle write along real runs. This file edits blobs
(at offsets from oracle.state_blob, the tests' own reading of the format) to reach what those runs never do:
- every check set_state makes before it writes anything. Each edited blob is loaded in a process of its own,
  which must exit with `fatal: set_state:` and a message naming the check;
- the reference's two readings of a stored bool: an entity's flags are read `!= 0`, a game's own bools `> 0`.
  The library must write back what the oracle writes back;
- what set_state keeps from the handle rather than the blob, on purpose: the per-VecGame constants,
  is_waiting_for_step, use_procgen_background, asset_rand_gen, and the entries of a vector past a short length."""
import os
import struct
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

import pytest

from helpers import make_pair
from level_seed_oracle import field_offsets
from oracle.ref_env import RefVecEnv, default_pack, mt19937_actions
from oracle.state_blob import ENTITY_FIELDS, parse

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KW = dict(distribution_mode="hard", num_levels=200, start_level=0, rand_seed=0)
PLAYER, BOSS, SHIELDS, GOAL = 0, 2, 3, 1  # entity types: pg_common.cuh, games/bossfight.cuh, games/jumper.cuh
LIST_WORDS, MAX_SPAWNERS = 400, 256       # games/chaser.cuh, games/starpilot.cuh
OTHER_TYPE = 99                            # an entity type no game uses


def lib_env(lib, game, n=4):
    return RefVecEnv(n, game, lib_path=lib, resource_root=default_pack(), **KW)


def state_after_steps(lib, game, steps=30):
    env = lib_env(lib, game)
    for a in mt19937_actions(1, env.num, steps):
        env.act(a)
    blob = env.get_state(1)
    env.close()
    return blob


def i32(blob, off):
    return struct.unpack_from("<i", blob, off)[0]


def ints(*values):
    return struct.pack(f"<{len(values)}i", *values)


def put(blob, off, *values):
    """blob with int32 values written from byte off on"""
    return blob[:off] + ints(*values) + blob[off + 4 * len(values):]


def splice(blob, off, old_bytes, new):
    return blob[:off] + new + blob[off + old_bytes:]


def tail(blob):
    return parse(blob)["tail_offset"]


def n_ents_at(blob):
    return field_offsets(blob)["grid_size"][0] + 4


def entity_field_at(blob, i, field):
    return n_ents_at(blob) + 4 + 4 * (i * len(ENTITY_FIELDS) + [f for f, _ in ENTITY_FIELDS].index(field))


def after_entities(blob):
    """offset of use_procgen_background"""
    return entity_field_at(blob, len(parse(blob)["entities"]), "x")


def asset_rand_gen_at(blob):
    return after_entities(blob) + 4 * 19  # use_procgen_background .. step_rand_int


def grid_w_at(blob):
    return tail(blob) - 4 * len(parse(blob)["grid"]) - 12


def retype(blob, old, new):
    """blob with every entity of type old given type new"""
    for i, ent in enumerate(parse(blob)["entities"]):
        if ent["type"] == old:
            blob = put(blob, entity_field_at(blob, i, "type"), new)
    return blob


def plunder_length_at(blob, vector):
    t = tail(blob)
    lanes = i32(blob, t + 4)
    return {"lane_directions": t + 4, "target_bools": t + 8 + 4 * lanes, "image_permutation": t + 12 + 4 * lanes + 24,
            "lane_vels": t + 16 + 4 * lanes + 48}[vector]


# case: (game, edit of a blob of that game, what the fatal message names)
REJECTIONS = {
    "version": ("coinrun", lambda b: put(b, 0, 1), "version"),
    "game_name": ("coinrun", lambda b: b.replace(b"coinrun", b"bigfish", 1), "another game"),
    "use_generated_assets": ("coinrun", lambda b: put(b, field_offsets(b)["use_generated_assets"][0], 1), "use_generated_assets"),
    "entity_count": ("coinrun", lambda b: put(b, n_ents_at(b), 1 << 20), "entities"),
    "grid_width": ("coinrun", lambda b: put(b, grid_w_at(b), i32(b, grid_w_at(b)) + 1), "grid"),
    "cut_short": ("coinrun", lambda b: b[:-8], "truncated"),
    "end_marker": ("coinrun", lambda b: put(b, len(b) - 4, 0), "trailing bytes"),
    "no_agent": ("coinrun", lambda b: retype(b, PLAYER, OTHER_TYPE), "agent"),
    "attack_modes": ("bossfight", lambda b: put(b, tail(b), 9), "attack_modes"),
    "free_cells": ("chaser", lambda b: put(b, tail(b), LIST_WORDS + 1), "free_cells"),
    "is_space_vec": ("chaser", lambda b: put(b, tail(b) + 4 + 4 * i32(b, tail(b)), LIST_WORDS + 1), "is_space_vec"),
    "has_keys": ("heist", lambda b: put(b, tail(b) + 8, 5), "has_keys"),
    "has_keys_negative": ("heist", lambda b: put(b, tail(b) + 8, -1), "has_keys"),
    "road_lane_speeds": ("leaper", lambda b: put(b, tail(b) + 4, 9), "road_lane_speeds"),
    "water_lane_speeds": ("leaper", lambda b: put(b, tail(b) + 12 + 4 * i32(b, tail(b) + 4), 9), "water_lane_speeds"),
    "lane_directions": ("plunder", lambda b: put(b, plunder_length_at(b, "lane_directions"), 6), "lane_directions"),
    "target_bools": ("plunder", lambda b: put(b, plunder_length_at(b, "target_bools"), 7), "target_bools"),
    "image_permutation": ("plunder", lambda b: put(b, plunder_length_at(b, "image_permutation"), 7), "image_permutation"),
    "lane_vels": ("plunder", lambda b: put(b, plunder_length_at(b, "lane_vels"), 6), "lane_vels"),
    "spawners": ("starpilot", lambda b: put(b, tail(b), MAX_SPAWNERS + 1), "spawner"),
    "no_boss": ("bossfight", lambda b: retype(b, BOSS, OTHER_TYPE), "boss"),
    "no_shields": ("bossfight", lambda b: retype(b, SHIELDS, OTHER_TYPE), "shields"),
    "no_goal": ("jumper", lambda b: retype(b, GOAL, OTHER_TYPE), "goal"),
}

SET_STATE = r"""
import sys
sys.path.insert(0, {root!r})
from oracle.ref_env import RefVecEnv, default_pack
env = RefVecEnv(1, {game!r}, lib_path={lib!r}, resource_root=default_pack(), **{kw!r})
env.set_state(0, open({path!r}, "rb").read())
print("set_state returned")
"""


@pytest.fixture(scope="module")
def rejected(hostsim_lib, tmp_path_factory):
    """{case: (exit code, stderr)} of one set_state of each REJECTIONS blob, each in a process of its own
    (set_state's refusal is fatal)"""
    blobs = {game: state_after_steps(hostsim_lib, game) for game in sorted({g for g, _, _ in REJECTIONS.values()})}
    d = tmp_path_factory.mktemp("blobs")
    for case, (game, edit, _) in REJECTIONS.items():
        edited = edit(blobs[game])
        assert edited != blobs[game], f"{case}: the edit changed nothing"
        (d / case).write_bytes(edited)

    def run(case):
        script = SET_STATE.format(root=ROOT, game=REJECTIONS[case][0], lib=hostsim_lib, kw=KW, path=str(d / case))
        r = subprocess.run([sys.executable, "-c", script], capture_output=True, text=True, timeout=300)
        return r.returncode, r.stdout + r.stderr

    with ThreadPoolExecutor(max_workers=os.cpu_count() or 4) as ex:
        return dict(zip(REJECTIONS, ex.map(run, REJECTIONS)))


@pytest.mark.parametrize("case", list(REJECTIONS))
def test_set_state_refuses_a_bad_blob(rejected, case):
    code, out = rejected[case]
    fatal = [line for line in out.splitlines() if line.startswith("fatal: set_state:")]
    assert code != 0 and fatal, out[-2000:]
    assert REJECTIONS[case][2] in fatal[0], fatal[0]


def test_bools_read_back_as_the_oracle_reads_them(ref_lib, hostsim_lib):
    """Two entity flags set to 2 and -1 both read as set; coinrun's has_support at -1 reads as clear and
    facing_right at 2 as set. The oracle and the library write back the same blob."""
    blob = state_after_steps(hostsim_lib, "coinrun")
    edited = put(blob, entity_field_at(blob, 0, "collides_with_entities"), 2)
    edited = put(edited, entity_field_at(edited, 1, "auto_erase"), -1)
    edited = put(edited, tail(edited) + 8, -1, 2)  # has_support, facing_right
    ref, dut = make_pair(hostsim_lib, 2, "coinrun", **dict(KW, rand_seed=5))
    ref.set_state(0, edited)
    dut.set_state(0, edited)
    out = ref.get_state(0)
    assert dut.get_state(0) == out
    ents = parse(out)["entities"]
    assert (ents[0]["collides_with_entities"], ents[1]["auto_erase"]) == (1, 1)
    assert struct.unpack_from("<2i", out, tail(out) + 8) == (0, 1)
    ref.close()
    dut.close()


def test_set_state_keeps_the_handles_own_fields(hostsim_lib):
    """The reference takes these from the blob; the library keeps the handle's per-VecGame constants, writes 0 for
    is_waiting_for_step and use_procgen_background and the default engine for asset_rand_gen. So get_state gives
    back the blob as it was before the edit."""
    env = lib_env(hostsim_lib, "coinrun")
    for a in mt19937_actions(1, env.num, 30):
        env.act(a)
    blob = env.get_state(1)
    offs = field_offsets(blob)
    edited = blob
    for k in ("use_easy_jump", "plain_assets", "physics_mode", "game_type", "is_waiting_for_step"):
        edited = put(edited, offs[k][0], i32(blob, offs[k][0]) + 1)
    edited = put(edited, after_entities(edited), 1)
    a = asset_rand_gen_at(edited)
    seeded, text = parse(blob)["rand_gen"]
    edited = splice(edited, a, 8 + i32(edited, a + 4), ints(seeded, len(text)) + text)
    p, q = parse(blob), parse(edited)
    assert [k for k in p if k != "tail_offset" and p[k] != q[k]] == ["use_easy_jump", "plain_assets", "physics_mode", "game_type",
                                                                     "is_waiting_for_step", "use_procgen_background", "asset_rand_gen"]
    env.set_state(1, edited)
    assert env.get_state(1) == blob
    env.close()


def test_short_vectors_keep_the_envs_entries(hostsim_lib):
    """A vector the blob gives fewer entries than the env has (plunder's target_bools, heist's has_keys) sets those
    entries only: get_state writes the length the env has (6, num_keys), the entries past the blob's length as the
    env held them."""
    env = lib_env(hostsim_lib, "plunder", n=1)
    blob = env.get_state(0)
    at = plunder_length_at(blob, "target_bools")
    ones = put(blob, at + 4, *[1] * 6)
    env.set_state(0, ones)
    assert env.get_state(0) == ones
    env.set_state(0, splice(ones, at, 4 + 4 * 6, ints(3, 0, 0, 0)))
    assert env.get_state(0) == put(ones, at + 4, 0, 0, 0)
    env.close()

    env = lib_env(hostsim_lib, "heist", n=1)
    blob = env.get_state(0)
    t = tail(blob)  # num_keys, world_dim, has_keys' length, has_keys
    three = splice(put(blob, t, 3), t + 8, 4 + 4 * i32(blob, t + 8), ints(3, 1, 1, 1))
    env.set_state(0, three)
    assert env.get_state(0) == three
    env.set_state(0, splice(three, t + 8, 4 + 4 * 3, ints(2, 0, 0)))
    assert env.get_state(0) == put(three, t + 12, 0, 0)
    env.close()
