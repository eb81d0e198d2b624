"""What the pause mask (pgb200_get_pause_mask) costs and saves.

1. Step time: per configuration, a handle without the mask and one with it, the mask holding a fixed random 0 %, 50 %,
   90 % and 99 % of the envs. After a desynchronising rollout, timed windows alternate; per window the device time
   per step (CUDA events on the stepping stream) and the running env-steps/s (envs not paused x steps / time).
2. One-episode-per-level evaluation: `--eval-envs` held-out levels of `--eval-game` (seeds from 10**9 on, outside
   the training range), each env put on its level with next_level_seeds() and action -1, then a uniform random
   policy until every env's first episode has ended (final_outputs()["level_end"] != 0). With pausing, an env is
   paused from the step after its episode ended; without it, ended envs keep playing until the last level ends.
   Wall-clock time of each (two runs each, alternating) and the steps taken.
One JSON line per measurement, with the card's name, power limit and maximum SM clock read in the same process.

usage: python tools/pause_bench.py [--steps 200] [--rounds 3] [--desync 200] [game:mode:envs ...]
"""
import argparse
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from tools.graph_step_bench import card  # noqa: E402

FRACTIONS = (0.0, 0.5, 0.9, 0.99)


def step_time(torch, ProcgenGym3Env, game, mode, n, args, info):
    gen = torch.Generator(device="cuda").manual_seed(1234)
    T = 256
    actions = torch.randint(0, 15, (T, n), device="cuda", dtype=torch.int32, generator=gen)
    kinds = ["no_mask"] + [f"paused_{int(f * 100)}pct" for f in FRACTIONS]
    envs = {k: ProcgenGym3Env(n, game, distribution_mode=mode, num_levels=0, start_level=0, rand_seed=0) for k in kinds}
    running = {"no_mask": n}
    for f, k in zip(FRACTIONS, kinds[1:]):
        m = torch.zeros(n, dtype=torch.uint8, device="cuda")
        m[torch.randperm(n, device="cuda", generator=gen)[:int(round(f * n))]] = 1
        running[k] = n - int(m.sum())
        envs[k].pause_mask().copy_(m)
    state = dict.fromkeys(kinds, 0)

    def run(k, steps):
        for t in range(state[k], state[k] + steps):
            envs[k].act(actions[t % T])
        state[k] += steps

    # the desynchronising rollout runs unpaused, so that every handle starts its windows from the same kind of states
    for k in kinds:
        m = envs[k].pause_mask().clone() if k != "no_mask" else None
        if m is not None:
            envs[k].pause_mask().zero_()
        run(k, args.desync)
        if m is not None:
            envs[k].pause_mask().copy_(m)
    torch.cuda.synchronize()
    ms = {k: [] for k in kinds}
    for r in range(args.rounds):
        for k in (kinds if r % 2 == 0 else kinds[::-1]):
            ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            ev0.record()
            run(k, args.steps)
            ev1.record()
            torch.cuda.synchronize()
            ms[k].append(ev0.elapsed_time(ev1) / args.steps)
    out = {"measure": "step_time", "config": f"{game} {mode} x{n}", "card": info, "steps_per_window": args.steps,
           "ms_per_step": ms, "running_envs": running,
           "running_env_steps_per_s": {k: [running[k] / (v / 1e3) for v in ms[k]] for k in kinds},
           "errors": {k: envs[k].errors() for k in kinds}}
    print(json.dumps(out), flush=True)
    for e in envs.values():
        e.close()


def evaluation(torch, ProcgenGym3Env, game, mode, n, info, pause, seed):
    env = ProcgenGym3Env(n, game, distribution_mode=mode, num_levels=0, start_level=0, rand_seed=seed)
    levels = torch.arange(n, device="cuda", dtype=torch.int32) + 10 ** 9
    env.next_level_seeds().copy_(levels)
    level_end = env.final_outputs()["level_end"]
    mask = env.pause_mask() if pause else None
    gen = torch.Generator(device="cuda").manual_seed(seed)
    env.act(torch.full((n,), -1, dtype=torch.int32, device="cuda"))
    assert torch.equal(env.get_info_tensors()["level_seed"], levels)
    done = torch.zeros(n, dtype=torch.bool, device="cuda")
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    steps = 0
    env_steps = torch.zeros((), dtype=torch.int64, device="cuda")
    while True:
        a = torch.randint(0, 15, (n,), device="cuda", dtype=torch.int32, generator=gen)
        if pause:
            mask.copy_(done.to(torch.uint8))
        env_steps += (~done).sum() if pause else n
        env.act(a)
        done |= level_end != 0
        steps += 1
        if steps % 16 == 0 and bool(done.all()):
            break
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0
    out = {"measure": "evaluation", "config": f"{game} {mode} x{n}", "pause": pause, "card": info, "wall_s": wall,
           "steps": steps, "env_steps_simulated": int(env_steps), "errors": env.errors()}
    env.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200, help="steps per timed window")
    ap.add_argument("--rounds", type=int, default=3, help="timed windows per handle, alternating")
    ap.add_argument("--desync", type=int, default=200)
    ap.add_argument("--eval-game", default="heist:hard")
    ap.add_argument("--eval-envs", type=int, default=32768)
    ap.add_argument("configs", nargs="*", default=["coinrun:easy:65536", "bigfish:hard:65536"])
    args = ap.parse_args()

    import torch

    from procgen_b200 import ProcgenGym3Env

    if not torch.cuda.is_available():
        raise SystemExit("pause_bench needs a CUDA device")
    torch.cuda.set_device(0)
    info = card()
    for cfg in args.configs:
        game, mode, n = cfg.split(":")
        step_time(torch, ProcgenGym3Env, game, mode, int(n), args, info)
    game, mode = args.eval_game.split(":")
    for r in range(2):
        for pause in ((True, False) if r % 2 == 0 else (False, True)):
            print(json.dumps(evaluation(torch, ProcgenGym3Env, game, mode, args.eval_envs, info, pause, seed=r)), flush=True)


if __name__ == "__main__":
    main()
