"""Device time of one snapshot apply (env.apply_snapshots()) against get_state / set_state of the same envs on the same
handle. For each configuration, after 60 device-resident steps (num_levels = 0), CUDA events time one apply that
  - saves every env (save_from = every env, one slot each),
  - loads every env (load_from = every env, from its own slot),
  - clones a random half (a random half of the slots save their env again; a random half of the envs load a random
    slot of their own game),
  - loads 1 % of the envs (random envs, random slots of their own game),
each the median of `--repeats` applies (the arrays refilled by torch before each, outside the timed window), and the
wall time of get_state() / set_state(blobs) of every env once. Checks that a load gives the blob get_state gave the
source. Prints one JSON line per configuration, with the card's name and power limit read in the same run.

    python tools/snapshot_bench.py [--repeats 10] [--out RESULTS.json]
"""
import argparse
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

ALL16 = "bigfish,bossfight,caveflyer,chaser,climber,coinrun,dodgeball,fruitbot,heist,jumper,leaper,maze,miner,ninja,plunder,starpilot"
CONFIGS = [("coinrun", "easy", 65536, 1), (ALL16, "hard", 32768, 16)]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def run(name, mode, n, games, repeats):
    import torch

    from procgen_b200 import ProcgenGym3Env

    env = ProcgenGym3Env(n, name, distribution_mode=mode, num_levels=0, start_level=0, rand_seed=0, resource_root=STANDIN_PACK)
    acts = mt19937_actions(0, n, 60)
    for t in range(60):
        env.act(torch.as_tensor(acts[t], device="cuda"))
    st = env.snapshots(n)
    everyone = torch.arange(n, dtype=torch.int32, device="cuda")
    rng = np.random.RandomState(0)
    st["save_from"].copy_(everyone)
    env.apply_snapshots()  # every slot holds its env: the loads below always find a state of their game
    t0 = time.perf_counter()
    blobs = env.get_state()
    t_get = time.perf_counter() - t0
    # env e takes the state of env e + games (same game), saved with the blobs
    st["load_from"].copy_((everyone + games) % n)
    env.apply_snapshots()
    sample = list(range(0, n, 61))
    assert env.get_state(sample) == [blobs[(e + games) % n] for e in sample], "a load differs from its source's blob"

    def same_game_slots(envs):
        # slot s holds env s after the first apply: a slot of env e's game is e % games + games * k
        k = rng.randint(0, n // games, size=len(envs))
        return torch.as_tensor(envs % games + games * k, dtype=torch.int32, device="cuda")

    def half_clone():
        save = torch.full((n,), -1, dtype=torch.int32, device="cuda")
        picks = torch.as_tensor(rng.permutation(n)[: n // 2], device="cuda")
        save[picks] = picks.to(torch.int32)  # slot p saves env p again
        load = torch.full((n,), -1, dtype=torch.int32, device="cuda")
        envs = rng.permutation(n)[: n // 2]
        load[torch.as_tensor(envs, device="cuda")] = same_game_slots(envs)
        return save, load

    def one_percent():
        load = torch.full((n,), -1, dtype=torch.int32, device="cuda")
        envs = rng.permutation(n)[: n // 100]
        load[torch.as_tensor(envs, device="cuda")] = same_game_slots(envs)
        return None, load

    cases = {
        "save_all": lambda: (everyone, None),
        "load_all": lambda: (None, everyone),
        "clone_half": half_clone,
        "load_1pct": one_percent,
    }
    ms = {}
    for case, make in cases.items():
        times = []
        for _ in range(repeats):
            save, load = make()
            st["save_from"].copy_(save if save is not None else torch.full_like(st["save_from"], -1))
            st["load_from"].copy_(load if load is not None else torch.full_like(st["load_from"], -1))
            start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            start.record()
            env.apply_snapshots()
            stop.record()
            stop.synchronize()
            times.append(start.elapsed_time(stop))
            assert int((st["load_from"] >= 0).sum()) == 0 and int((st["save_from"] >= 0).sum()) == 0, case
        ms[case] = round(float(np.median(times)), 3)
    t0 = time.perf_counter()
    env.set_state(blobs)
    torch.cuda.synchronize()
    t_set = time.perf_counter() - t0
    res = dict(game="all16" if games > 1 else name, mode=mode, envs=n, card=card(), apply_ms=ms,
               get_state_all_s=round(t_get, 3), set_state_all_s=round(t_set, 3), errors=env.errors())
    env.close()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=10)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    results = []
    for name, mode, n, games in CONFIGS:
        r = run(name, mode, n, games, args.repeats)
        print(json.dumps(r), flush=True)
        results.append(r)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        json.dump(results, open(args.out, "w"), indent=1)


if __name__ == "__main__":
    main()
