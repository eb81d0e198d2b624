"""Per-env logic-kernel duration at steady state, split into steps that ended an episode (level
generation) and ordinary steps. Needs PGB200_DEBUG_TIMING=1 (set here). One JSON line per game.
usage: python tools/gpu_reset_cost.py [--num-levels L] [--bank] [envs] [desync_steps] [game:mode ...]
--num-levels L plays the levels [0, L) (default 0: unboundedly many); --bank also banks them (build_level_bank)."""
import json
import os
import sys

os.environ["PGB200_DEBUG_TIMING"] = "1"
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from procgen_b200 import ENV_NAMES, ProcgenGym3Env

args = sys.argv[1:]
num_levels, bank = 0, "--bank" in args
if "--num-levels" in args:
    i = args.index("--num-levels")
    num_levels = int(args[i + 1])
    del args[i:i + 2]
args = [a for a in args if a != "--bank"]
n = int(args[0]) if len(args) > 0 else 32768
desync = int(args[1]) if len(args) > 1 else 600
games = args[2:] or [g + ":hard" for g in ENV_NAMES]
for gm in games:
    game, mode = gm.split(":")
    env = ProcgenGym3Env(n, game, distribution_mode=mode, num_levels=num_levels, rand_seed=0)
    if bank:
        env.build_level_bank()
    g = torch.Generator(device="cuda").manual_seed(0)
    acts = torch.randint(0, 15, (64, n), device="cuda", dtype=torch.int32, generator=g)
    for t in range(desync):
        env.act(acts[t % 64])
    env.set_launch_shape(chunks=1, serialize=True)
    cyc = np.zeros(n, np.uint32)
    r_c, n_c = [], []
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    env.kernel_timing_begin(64)
    for t in range(16):
        env.act(acts[t])
        rew, ob, first = env.observe()
        torch.cuda.synchronize()
        assert env._lib.pgb200_debug_cycles(env._h, cyc.ctypes.data) == 0
        f = first.cpu().numpy()
        r_c.append(cyc[f].astype(np.float64))
        n_c.append(cyc[~f].astype(np.float64))
    kt = env.kernel_timing_end()
    r = np.concatenate(r_c)
    q = np.concatenate(n_c)
    out = {"game": game, "mode": mode, "envs": n, "num_levels": num_levels, "bank": bank, "resets_per_step": len(r) / 16.0,
           "reset_cycles": {"mean": float(r.mean()) if len(r) else None, "p50": float(np.percentile(r, 50)) if len(r) else None,
                            "p99": float(np.percentile(r, 99)) if len(r) else None, "max": float(r.max()) if len(r) else None},
           "step_cycles": {"mean": float(q.mean()), "p50": float(np.percentile(q, 50)), "p99": float(np.percentile(q, 99)), "max": float(q.max())},
           "reset_share_of_cycles": float(r.sum() / (r.sum() + q.sum())) if len(r) else 0.0,
           "logic_ms": kt["logic_ms"] / max(1, kt["launch_pairs"]), "render_ms": kt["render_ms"] / max(1, kt["launch_pairs"]),
           "errors": env.errors()}
    print(json.dumps(out), flush=True)
    env.close()
