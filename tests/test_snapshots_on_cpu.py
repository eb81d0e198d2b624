"""Snapshot slots (pgb200_get_snapshots / pgb200_apply_snapshots) in the host debug build.

A load must make an env a byte-for-byte copy of its source at save time, and an apply must touch nothing else. Each case
therefore runs three handles of the build under test on the same actions: `dut` saves and loads; `twin` receives the
same states through set_states; `control` never changes. After the loads, dut's loaded envs must hold their source's
save-time header, live entities and blob, and dut and twin then run in lockstep for 50 steps, outputs and blobs
compared every step, with dut's other envs checked against the control.

Covered: all 16 games easy and hard, the extreme and memory modes, the 16-game list, the whole-world view and
sequential levels; a load into the env saved, into another env, from one slot into several envs, and into an env saved
in the same call; the entries an apply refuses; every opt-in of the step; the kernel launches of one apply."""
import zlib

import numpy as np
import pytest

from helpers import read_lib_array
from level_bank import bank_info, build_bank
from level_lookahead import enable_lookahead, lookahead_info
from level_seed_oracle import next_level_seeds
from oracle.ref_env import RefVecEnv, default_pack, mt19937_actions
from pause_oracle import pause_mask
from rollout import get_rollout, snapshot
from snapshots import apply, assert_same, get_snapshots, launches, observation, read_env, same_game
from state_batch import get_states, set_states
from test_state_batch_on_cpu import ALL16, CASES, _final_outputs, _id


def _handles(lib, n, name, kw, count=3):
    return [RefVecEnv(n, name, lib_path=lib, resource_root=default_pack(), **kw) for _ in range(count)]


def _step(envs, a):
    for env in envs:
        env.act(a)


@pytest.mark.parametrize("case", CASES, ids=[_id(c) for c in CASES])
def test_loads_are_exact_copies(hostsim_lib, case):
    name, mode, extra = case
    games = 16 if name == ALL16 else 1
    n = 32 if name == ALL16 else 6
    kw = dict(distribution_mode=mode, num_levels=200, start_level=0, rand_seed=0, **extra)
    dut, twin, control = handles = _handles(hostsim_lib, n, name, kw)
    rng = np.random.RandomState(zlib.crc32(_id(case).encode()))
    acts = mt19937_actions(0, n, 70)
    for t in range(12):
        _step(handles, acts[t])
    rc, st = get_snapshots(dut, 4)
    assert rc == 0
    # three envs saved into slots 0-2; in the list, consecutive envs of three different games
    if games > 1:
        e0 = int(rng.randint(n))
        a = [(e0 + k) % n for k in range(3)]
    else:
        a = [int(e) for e in rng.permutation(n)[:3]]
    st["save_from"][:3] = a
    saved_blobs = get_states(dut, a)
    saved_env = [read_env(dut, e) for e in a]
    assert apply(dut) == 0
    assert (st["save_from"] == [-1, -1, -1, -1]).all() and (st["source"] == a + [-1]).all()
    assert get_states(dut, list(range(n))) == get_states(twin, list(range(n))), "a save changed an env"
    for t in range(12, 17):
        _step(handles, acts[t])
    # the loads: a[0] from its own slot; another env of a[1]'s game from slot 1; two envs of a[2]'s game from slot 2,
    # one of which (y) is also saved into slot 3 in the same call
    b1 = same_game(n, games, a[1], exclude=a)[0]
    many = same_game(n, games, a[2], exclude=[a[0], b1])[:2]
    y = many[0]
    y_blob = get_states(dut, [y])[0]
    st["load_from"][[a[0], b1] + many] = [0, 1, 2, 2]
    st["save_from"][3] = y
    loaded = {a[0]: 0, b1: 1, many[0]: 2, many[1]: 2}
    assert apply(dut) == 0
    assert (st["load_from"] == -1).all() and (st["save_from"] == -1).all() and st["source"][3] == y
    for e, s in loaded.items():
        assert read_env(dut, e) == saved_env[s], f"env {e}: header or entities differ from slot {s}'s source at save time"
    assert get_states(dut, list(loaded)) == [saved_blobs[s] for s in loaded.values()]
    # slot 3 holds y as it was before the call: load it back
    st["load_from"][y] = 3
    assert apply(dut) == 0 and st["load_from"][y] == -1
    loaded[y] = 3
    final_blobs = get_states(dut, list(loaded))
    assert final_blobs == [saved_blobs[s] if s < 3 else y_blob for s in loaded.values()]
    assert set_states(twin, list(loaded), final_blobs) == 0
    rest = np.setdiff1d(np.arange(n), list(loaded))
    assert_same(observation(dut), observation(twin), np.arange(n), "after the loads")
    for t in range(17, 67):
        _step(handles, acts[t])
        out = observation(dut)
        assert_same(out, observation(twin), np.arange(n), f"step {t}")
        assert_same(out, observation(control), rest, f"step {t}, envs not loaded")
        blobs = get_states(dut, list(range(n)))
        assert blobs == get_states(twin, list(range(n))), f"step {t}: blobs differ"
        assert [blobs[e] for e in rest] == get_states(control, rest), f"step {t}: an env not loaded changed"
    for env in handles:
        env.close()


def test_refused_entries_stay_and_change_nothing(hostsim_lib):
    """In the 16-game list: envs and slots out of range, an empty slot and a slot holding another game's state. Every
    refused entry keeps the value written, and no env, output or slot changes; the accepted entries of the same call
    are applied."""
    n, games = 32, 16
    kw = dict(distribution_mode="hard", num_levels=0, rand_seed=0)
    dut, twin = handles = _handles(hostsim_lib, n, ALL16, kw, count=2)
    for a in mt19937_actions(0, n, 8):
        _step(handles, a)
    rc, st = get_snapshots(dut, 3)
    assert rc == 0
    st["save_from"][:] = [0, n, -7]  # env 0 (game 0) into slot 0; the others refused
    before = get_states(dut, [0])
    assert apply(dut) == 0
    assert list(st["save_from"]) == [-1, n, -7] and list(st["source"]) == [0, -1, -1]
    obs, blobs = observation(dut), get_states(dut, list(range(n)))
    # 1 plays game 1 (slot 0 holds game 0); slots 1 and 3, 99 are empty or out of range; 16 plays game 0: accepted
    st["load_from"][[1, 2, 3, 4, 16]] = [0, 1, 3, 99, 0]
    st["save_from"][1] = 12345
    assert apply(dut) == 0
    assert list(st["load_from"][[1, 2, 3, 4, 16]]) == [0, 1, 3, 99, -1]
    assert list(st["save_from"]) == [-1, 12345, -7] and list(st["source"]) == [0, -1, -1]
    others = [e for e in range(n) if e != 16]
    assert_same(observation(dut), obs, others, "refused loads")
    now = get_states(dut, list(range(n)))
    assert [now[e] for e in others] == [blobs[e] for e in others], "a refused entry changed an env"
    assert now[16] == before[0]
    assert set_states(twin, [16], before) == 0
    for a in mt19937_actions(1, n, 10):
        _step(handles, a)
        assert_same(observation(dut), observation(twin), np.arange(n), "after the refusals")
    for env in handles:
        env.close()


def test_every_opt_in(hostsim_lib):
    """Final outputs, the rollout, the pause mask, pending overrides, a bank of half the level set and level lookahead
    on dut and twin alike. An apply that saves and loads envs, paused ones among them, writes none of the opt-ins' arrays
    (the overrides are neither read nor consumed) and the loaded paused envs stay paused; then lockstep with the twin
    (which received the same states through set_states) through forced resets, in which the lookahead slots of the
    loaded envs miss once, then serve."""
    n, name = 8, "coinrun"
    kw = dict(distribution_mode="hard", num_levels=50, start_level=0, rand_seed=0)
    dut, twin = handles = _handles(hostsim_lib, n, name, kw, count=2)
    opt = []
    for env in handles:
        final = _final_outputs(env)
        rc, roll = get_rollout(env, 4)
        assert rc == 0
        mask, seeds = pause_mask(env), next_level_seeds(env)
        assert build_bank(env, range(0, 25)) == 0 and enable_lookahead(env) == 0
        opt.append((final, roll, mask, seeds))
    acts = mt19937_actions(0, n, 90)
    for t in range(20):
        _step(handles, acts[t])
    rc, st = get_snapshots(dut, 4)
    assert rc == 0
    st["save_from"][:] = [6, 0, 3, 7]
    saved = get_states(dut, [6, 0, 3, 7])
    assert apply(dut) == 0
    for t in range(20, 30):
        _step(handles, acts[t])
    paused = np.zeros(n, np.uint8)
    paused[[1, 2, 5]] = 1
    for final, roll, mask, seeds in opt:
        mask[:] = paused
        seeds[:] = 7
    final, roll, mask, seeds = opt[0]
    before = {"final": {k: read_lib_array(v) for k, v in final.items()}, "roll": snapshot(roll), "bank": bank_info(dut),
              "look": lookahead_info(dut)}
    loads = {5: 0, 2: 1, 1: 2, 4: 3, 7: 3}  # paused 5, 2, 1 among them
    for e, s in loads.items():
        st["load_from"][e] = s
    assert apply(dut) == 0
    assert (read_lib_array(seeds) == 7).all() and np.array_equal(read_lib_array(mask), paused)
    for k, v in final.items():
        assert np.array_equal(read_lib_array(v), before["final"][k]), f"apply changed the final outputs' {k}"
    for k, v in snapshot(roll).items():
        assert np.array_equal(v, before["roll"][k]), f"apply changed the rollout's {k}"
    assert bank_info(dut) == before["bank"] and lookahead_info(dut) == before["look"]
    blobs = get_states(dut, list(loads))
    assert blobs == [saved[s] for s in loads.values()]
    assert set_states(twin, list(loads), blobs) == 0
    assert_same(observation(dut), observation(twin), np.arange(n), "after the loads")
    for e in opt:
        e[3][:] = -1
    for t in range(30, 35):
        _step(handles, acts[t])
        assert_same(observation(dut), observation(twin), np.arange(n), f"step {t}")
        assert get_states(dut, [5, 2, 1]) == [saved[0], saved[1], saved[2]], f"step {t}: a paused loaded env moved"
    for final, roll, mask, seeds in opt:
        mask[:] = 0
    look0 = lookahead_info(dut)
    for t in range(35, 90):
        a = acts[t].copy()
        if t % 8 == 0:
            a[:] = -1
        _step(handles, a)
        assert_same(observation(dut), observation(twin), np.arange(n), f"step {t}")
        for k in ("rgb", "level_end"):
            assert np.array_equal(read_lib_array(opt[0][0][k]), read_lib_array(opt[1][0][k])), f"step {t}: final {k}"
        assert all(np.array_equal(x, y) for x, y in zip(snapshot(opt[0][1]).values(), snapshot(opt[1][1]).values())), f"step {t}: rollout"
        assert get_states(dut, list(range(n))) == get_states(twin, list(range(n))), f"step {t}: blobs differ"
    look = lookahead_info(dut)
    assert look["generated"] > look0["generated"] and look["served"] > look0["served"], (look0, look)
    assert look == lookahead_info(twin)
    for env in handles:
        env.close()


@pytest.mark.parametrize("name", ["coinrun", ALL16])
def test_launches_of_one_apply(hostsim_lib, name):
    """pgb200_kernel_launches counts 2 + 2 G per apply (G games in the list), whatever the arrays hold"""
    games = 16 if name == ALL16 else 1
    n = 2 * games
    env = _handles(hostsim_lib, n, name, dict(distribution_mode="hard", num_levels=0, rand_seed=0), count=1)[0]
    rc, st = get_snapshots(env, 2)
    assert rc == 0
    # loads from empty slots, saves only, then loads (in the list, half of them refused)
    for save, load in (([-1, -1], [1, 0]), ([0, 1], [-1, -1]), ([-1, -1], [0, 1])):
        st["save_from"][:] = save
        st["load_from"][:] = load * games
        k = launches(env)
        assert apply(env) == 0
        assert launches(env) - k == 2 + 2 * games
    env.close()
