"""Steady-state step throughput of several configurations in one process, with the centred view or the whole-world
view (center_agent=False) that bench.py does not cover: the scrolling games then draw up to 64x64 cells per frame
with their whole-world setup and render kernels (FULL_VIEW_CELLS).

Per configuration, bench.py's protocol for `value`: a desync rollout, then K timed steps through env.act() /
env.observe() between CUDA events; then K more steps with the kernels serialised and timed one by one (the
`roofline` kernel times). One JSON line per configuration. A/B two builds by running this once per library,
alternating, with PROCGEN_B200_LIB selecting the library.

usage: python tools/steady_bench.py [--whole-world] [--steps 60] [--desync 1500] game:mode:envs [game:mode:envs ...]
       (game may be "all16", the 16-game joint list)"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from bench import ALL16, timed_rollout
from procgen_b200 import ProcgenGym3Env


def run(game, mode, n, steps, desync, center_agent):
    env = ProcgenGym3Env(n, ALL16 if game == "all16" else game, distribution_mode=mode, num_levels=0, start_level=0,
                         rand_seed=0, center_agent=center_agent)
    gen = torch.Generator(device="cuda").manual_seed(1234)
    T = 256
    actions = torch.randint(0, 15, (T, n), device="cuda", dtype=torch.int32, generator=gen)
    env.observe()
    for t in range(desync):
        env.act(actions[t % T])
        env.observe()
    torch.cuda.synchronize()
    ms = timed_rollout(env, actions, desync, steps, torch.cuda.synchronize)
    env.set_launch_shape(chunks=1, serialize=True)
    env.kernel_timing_begin(steps * 64)
    for t in range(steps):
        env.act(actions[t % T])
        env.observe()
    kt = env.kernel_timing_end()
    errors = env.errors()
    env.close()
    pairs = max(1, kt["launch_pairs"])
    return {"game": game, "mode": mode, "envs": n, "center_agent": center_agent, "steps": steps, "desync_steps": desync,
            "value": n * steps / (ms / 1000.0), "unit": "env-steps/s", "ms_per_step": ms / steps,
            "logic_kernel_ms_avg": kt["logic_ms"] / pairs, "setup_kernel_ms_avg": kt["setup_ms"] / pairs,
            "render_kernel_ms_avg": kt["render_ms"] / pairs, "env_error_bits": errors}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("configs", nargs="+", help="game:mode:envs")
    ap.add_argument("--whole-world", action="store_true", help="center_agent=False")
    ap.add_argument("--steps", type=int, default=60)
    ap.add_argument("--desync", type=int, default=1500)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    lib = os.environ.get("PROCGEN_B200_LIB", "default")
    for cfg in args.configs:
        game, mode, n = cfg.split(":")
        r = run(game, mode, int(n), args.steps, args.desync, not args.whole_world)
        r["lib"] = os.path.basename(lib)
        print(json.dumps(r), flush=True)


if __name__ == "__main__":
    main()
