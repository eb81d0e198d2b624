"""Wall time of get_state / set_state for every env of a handle: a loop of one-env calls (get_state / set_state of the
C ABI, what a caller paid per env before the batched calls) against one batched call (pgb200_get_states /
pgb200_set_states through ProcgenGym3Env), and of restoring a random 10 % of the envs; plus the bytes a transfer moves
per env against the size of its blob. Checks that both ways give the same blobs. Prints one JSON line per
configuration, with the card's name and power limit read in the same run.

    python tools/state_batch_bench.py [--sizes 4096,65536] [--out RESULTS.json]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle.record import STANDIN_PACK  # noqa: E402
from oracle.ref_env import mt19937_actions  # noqa: E402
from oracle.state_blob import parse  # noqa: E402

CONFIGS = [("coinrun", "easy"), ("caveflyer", "hard")]
# the packed record of pg_kernels.cuh (StateSlot): EnvHdr | two MT19937 | Entity[n_ents] | int16 grid[cells] | scratch;
# a transfer also gathers each header once more to size the records, and moves one 32-byte StateSlot per env
ENV_HDR, MT, ENTITY, SLOT = 496, 2512, 128, 32


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def get_moved_bytes(blob):
    """bytes a get_state of this env moves between host and device: its env index and header to size the record, its
    StateSlot and its packed record (coinrun and caveflyer keep no persistent scratch words). A set_state moves that
    and the slot and restored record once more."""
    p = parse(blob)
    rec = ENV_HDR + 2 * MT + ENTITY * len(p["entities"]) + ((2 * len(p["grid"]) + 15) & ~15)
    return 4 + ENV_HDR + SLOT + rec


def timed(fn):
    t0 = time.perf_counter()
    out = fn()
    return time.perf_counter() - t0, out


def run(name, mode, n):
    import torch

    from procgen_b200 import ProcgenGym3Env
    from procgen_b200.env import MAX_STATE_SIZE

    kw = dict(distribution_mode=mode, num_levels=0, start_level=0, resource_root=STANDIN_PACK)
    env = ProcgenGym3Env(n, name, rand_seed=0, **kw)
    acts = mt19937_actions(0, n, 60)
    for t in range(60):
        env.act(torch.as_tensor(acts[t], device="cuda"))
    env.get_state([0])  # staging and first-call costs out of the timed windows
    lib, h = env._lib, env._h
    buf = C.create_string_buffer(MAX_STATE_SIZE)

    def loop_get():
        out = []
        for i in range(n):
            k = lib.get_state(h, i, buf, MAX_STATE_SIZE)
            out.append(buf.raw[:k])
        return out

    t_loop_get, loop_blobs = timed(loop_get)
    t_get, blobs = timed(env.get_state)
    assert blobs == loop_blobs, "batched and one-env blobs differ"
    other = ProcgenGym3Env(n, name, rand_seed=1, **kw)
    other.get_state([0])
    t_set, _ = timed(lambda: other.set_state(blobs))
    assert other.get_state() == blobs
    fresh = ProcgenGym3Env(n, name, rand_seed=2, **kw)
    fresh.get_state([0])

    def loop_set():
        for i in range(n):
            lib.set_state(fresh._h, i, blobs[i], len(blobs[i]))

    t_loop_set, _ = timed(loop_set)
    assert fresh.get_state() == blobs
    sub = np.random.RandomState(0).permutation(n)[: n // 10]
    donor = [blobs[e] for e in sub]
    t_sub, _ = timed(lambda: env.set_state(donor, envs=sub))
    sizes = np.array([len(b) for b in blobs])
    sample = blobs[:: max(1, n // 256)]
    res = dict(game=name, mode=mode, envs=n, card=card(),
               get_loop_s=round(t_loop_get, 4), get_batched_s=round(t_get, 4),
               set_loop_s=round(t_loop_set, 4), set_batched_s=round(t_set, 4), set_10pct_s=round(t_sub, 4),
               blob_bytes_mean=float(sizes.mean()),
               get_moved_bytes_mean=float(np.mean([get_moved_bytes(b) for b in sample])),
               set_moved_bytes_mean=float(np.mean([2 * get_moved_bytes(b) - ENV_HDR - 4 for b in sample])),
               errors=env.errors() | other.errors() | fresh.errors())
    for e in (env, other, fresh):
        e.close()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="4096,65536")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    results = []
    for n in [int(s) for s in args.sizes.split(",")]:
        for name, mode in CONFIGS:
            r = run(name, mode, n)
            print(json.dumps(r), flush=True)
            results.append(r)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        json.dump(results, open(args.out, "w"), indent=1)


if __name__ == "__main__":
    main()
