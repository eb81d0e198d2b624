"""The seeds whose freshly generated level is the fullest, for every (game, distribution mode) pair.

Oracle only, on the CPU. For every pair the reference accepts (game.cpp:56-66) the levels of seeds 0 .. N-1
are generated through the oracle (each env's state blob patched to current_level_seed = s,
episodes_remaining = 1, then one step with action -1: the same reset an override takes), and for each
quantity the TOP seeds with the largest value are kept:

  entities  live entities right after generation (the state blob's entity list)
  cells     grid cells (grid_w * grid_h; only where the world size changes with the seed)
  open      grid cells unlike the corner cell, which every generator leaves as border or outer wall: the
            extent of the maze, cave or rooms where a fixed-size world holds a layout of varying size

A quantity that is the same for every scanned seed is not data dependent and is left out. Ties go to the
smaller seed, so the output depends only on the oracle and the arguments. The result is the data fixture
tests/golden/level_extremes.json; tests/level_sweep.py's sweep_seeds() puts these seeds into every sweep,
so the fullest levels of each mode (the ones nearest the fixed capacities ENT_CAP, SCRATCH_WORDS,
MAX_VISIBLE_ENTS, MAX_ROT_BLITS) are always compared on the GPU.

    python tests/tools/level_extremes.py [--seeds N] [--jobs J] [--out PATH]
"""
import argparse
import json
import os
import sys
from multiprocessing import Pool

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from level_sweep import LEVEL_EXTREMES, PAIRS  # noqa: E402

SEEDS = 50000
TOP = 4
BATCH = 64


def level_sizes(blob):
    """(live entities, grid cells, open cells) of a state blob."""
    from level_seed_oracle import field_offsets
    from oracle.state_blob import ENTITY_FIELDS, Reader

    r = Reader(blob)
    r.o = field_offsets(blob)["grid_size"][0] + 4
    n_ents = r.i()
    r.o += n_ents * 4 * len(ENTITY_FIELDS)
    r.o += 4 * (2 + 3 + 3 + 8 + 3)   # background, char_dim, actions, physics floats, three ints
    r.i()
    r.s()                           # asset_rand_gen
    r.o += 4 * (3 + 6)
    w, h = r.i(), r.i()
    n_cells = r.i()
    grid = np.frombuffer(blob, "<i4", n_cells, r.o)
    return n_ents, w * h, int((grid != grid[0]).sum())


def scan(args):
    """{quantity: [[value, seed], ...]} for seeds 0 .. n_seeds-1 of one pair."""
    game, mode, n_seeds = args
    from level_seed_oracle import patch_fields
    from oracle.ref_env import RefVecEnv

    env = RefVecEnv(BATCH, game, distribution_mode=mode, num_levels=0, start_level=0, rand_seed=0)
    base = [env.get_state(e) for e in range(BATCH)]
    force = np.full(BATCH, -1, np.int32)
    vals = np.zeros((n_seeds, 3), np.int64)
    for b in range(0, n_seeds, BATCH):
        seeds = range(b, min(b + BATCH, n_seeds))
        for e, s in enumerate(seeds):
            env.set_state(e, patch_fields(base[e], current_level_seed=s, episodes_remaining=1))
        env.act(force)
        for e, s in enumerate(seeds):
            vals[s] = level_sizes(env.get_state(e))
    env.close()
    out = {}
    for q, name in enumerate(("entities", "cells", "open")):
        v = vals[:, q]
        if v.min() == v.max():
            continue
        order = np.lexsort((np.arange(n_seeds), -v))[:TOP]
        out[name] = [[int(v[s]), int(s)] for s in order]
    return f"{game}/{mode}", out


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--seeds", type=int, default=SEEDS)
    ap.add_argument("--jobs", type=int, default=os.cpu_count())
    ap.add_argument("--out", default=LEVEL_EXTREMES)
    a = ap.parse_args()
    with Pool(a.jobs) as pool:
        res = dict(pool.map(scan, [(g, m, a.seeds) for g, m in PAIRS], chunksize=1))
    doc = {"seeds_scanned": a.seeds, "top": TOP, "pairs": {k: res[k] for k in sorted(res)}}
    with open(a.out, "w") as f:
        json.dump(doc, f, indent=1, sort_keys=True)
        f.write("\n")


if __name__ == "__main__":
    main()
