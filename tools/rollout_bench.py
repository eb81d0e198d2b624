"""What the rollout (env.rollout()) saves in a PPO-style collection loop.

Per configuration, two device-resident handles of the same configuration step the same actions:
  copy     a step, then the learner's three copies of its outputs into rollout storage of T + 1 slots
           (obs_buf[t].copy_(rgb); rew_buf[t].copy_(rew); first_buf[t].copy_(first))
  rollout  a step with env.rollout(T + 1) on, which stores the same outputs into its ring from the render kernel
Timed windows alternate between the two; per window the device time per step (CUDA events on the stepping stream).
After the windows the copy loop's storage and the rollout's ring must be equal, slot for slot. Then one window per
handle under kernel timing gives the render kernel's ms per step. One JSON line per configuration, with the card's
name, power limit and maximum SM clock read in the same process.

usage: python tools/rollout_bench.py [--steps 160] [--rounds 3] [--warmup 64] [--T 16] [game:mode:envs ...]
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from tools.graph_step_bench import card  # noqa: E402

ALL16 = "bigfish,bossfight,caveflyer,chaser,climber,coinrun,dodgeball,fruitbot,heist,jumper,leaper,maze,miner,ninja,plunder,starpilot"
DEFAULT = ["coinrun:easy:65536", f"{ALL16}:hard:32768"]


def bench(torch, ProcgenGym3Env, game, mode, n, args, info):
    gen = torch.Generator(device="cuda").manual_seed(1234)
    A = 256
    actions = torch.randint(0, 15, (A, n), device="cuda", dtype=torch.int32, generator=gen)
    slots = args.T + 1
    kw = dict(distribution_mode=mode, num_levels=0, start_level=0, rand_seed=0)
    envs = {"copy": ProcgenGym3Env(n, game, **kw), "rollout": ProcgenGym3Env(n, game, **kw)}
    # the learner's storage, and the rollout (both hold the initial outputs in slot 0)
    obs_buf = torch.empty((slots, n, 64, 64, 3), dtype=torch.uint8, device="cuda")
    rew_buf = torch.empty((slots, n), dtype=torch.float32, device="cuda")
    first_buf = torch.empty((slots, n), dtype=torch.uint8, device="cuda")
    rew, ob, first = envs["copy"].observe()
    obs_buf[0].copy_(ob["rgb"])
    rew_buf[0].copy_(rew)
    first_buf[0].copy_(first)
    roll = envs["rollout"].rollout(slots)
    state = dict.fromkeys(envs, 0)

    def run(k, steps):
        env = envs[k]
        for t in range(state[k], state[k] + steps):
            env.act(actions[t % A])
            if k == "copy":
                rew, ob, first = env.observe()
                s = (t + 1) % slots
                obs_buf[s].copy_(ob["rgb"])
                rew_buf[s].copy_(rew)
                first_buf[s].copy_(first)
        state[k] += steps

    for k in envs:
        run(k, args.warmup)
    torch.cuda.synchronize()
    ms = {k: [] for k in envs}
    order = list(envs)
    for r in range(args.rounds):
        for k in order:
            ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            ev0.record()
            run(k, args.steps)
            ev1.record()
            torch.cuda.synchronize()
            ms[k].append(ev0.elapsed_time(ev1) / args.steps)
        order = order[1:] + order[:1]
    assert state["copy"] == state["rollout"]
    same = int(roll["cursor"].item()) == state["rollout"] % slots
    same = same and torch.equal(roll["rgb"], obs_buf) and torch.equal(roll["rew"], rew_buf) and torch.equal(roll["first"], first_buf)
    render = {}
    steps_t = min(args.steps, 64)
    for k in envs:
        envs[k].kernel_timing_begin(steps_t * 128)
        run(k, steps_t)
        kt = envs[k].kernel_timing_end()
        render[k] = kt["render_ms"] / steps_t
    ngames = len(game.split(","))
    out = {"config": f"{game if ngames == 1 else f'{ngames}-game list'} {mode} x{n} T={args.T}", "card": info,
           "steps_per_window": args.steps, "ms_per_step": ms,
           "env_steps_per_s": {k: [n / (v / 1e3) for v in ms[k]] for k in envs},
           "render_kernel_ms_per_step": render, "rollout_equals_copies": bool(same),
           "errors": {k: envs[k].errors() for k in envs}}
    print(json.dumps(out), flush=True)
    for e in envs.values():
        e.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=160, help="steps per timed window")
    ap.add_argument("--rounds", type=int, default=3, help="timed windows per handle, alternating")
    ap.add_argument("--warmup", type=int, default=64)
    ap.add_argument("--T", type=int, default=16, help="steps per rollout: the storage holds T + 1 slots")
    ap.add_argument("configs", nargs="*", default=DEFAULT)
    args = ap.parse_args()

    import torch

    from procgen_b200 import ProcgenGym3Env

    if not torch.cuda.is_available():
        raise SystemExit("rollout_bench needs a CUDA device")
    torch.cuda.set_device(0)
    info = card()
    for cfg in args.configs:
        game, mode, n = cfg.split(":")
        bench(torch, ProcgenGym3Env, game, mode, int(n), args, info)


if __name__ == "__main__":
    main()
