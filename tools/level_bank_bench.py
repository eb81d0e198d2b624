"""What the level bank (build_level_bank) saves.

Per configuration, a banked and an unbanked handle of the same configuration (num_levels levels from 0; the bank
holds exactly them). After a warm-up that spreads episode ends, timed windows alternate between the two; per window
the device time per step (CUDA events on the stepping stream) and env-steps/s. Also the bank's build time (host clock
around the call, which returns when the bank is built), its bytes per level and total bytes. The outputs of the two
handles are compared after every window: a bank must not change them. One JSON line per configuration, with the
card's name, power limit and maximum SM clock read in the same process.

usage: python tools/level_bank_bench.py [--steps 200] [--rounds 3] [--warmup 300] [game:mode:envs:num_levels ...]
"""
import argparse
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from tools.graph_step_bench import card  # noqa: E402

ALL16 = "bigfish,bossfight,caveflyer,chaser,climber,coinrun,dodgeball,fruitbot,heist,jumper,leaper,maze,miner,ninja,plunder,starpilot"
DEFAULT = [f"{g}:hard:32768:500" for g in ("caveflyer", "jumper", "leaper", "coinrun", "heist", "maze")] + \
          ["coinrun:easy:65536:200", f"{ALL16}:hard:32768:500"]


def bench(torch, ProcgenGym3Env, game, mode, n, levels, args, info):
    gen = torch.Generator(device="cuda").manual_seed(1234)
    T = 256
    actions = torch.randint(0, 15, (T, n), device="cuda", dtype=torch.int32, generator=gen)
    kw = dict(distribution_mode=mode, num_levels=levels, start_level=0, rand_seed=0)
    envs = {"no_bank": ProcgenGym3Env(n, game, **kw), "bank": ProcgenGym3Env(n, game, **kw)}
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    envs["bank"].build_level_bank()
    build_s = time.perf_counter() - t0
    bank = envs["bank"].level_bank_info()
    state = dict.fromkeys(envs, 0)

    def run(k, steps):
        for t in range(state[k], state[k] + steps):
            envs[k].act(actions[t % T])
        state[k] += steps

    for k in envs:
        run(k, args.warmup)
    torch.cuda.synchronize()
    ms = {k: [] for k in envs}
    same = True
    for r in range(args.rounds):
        for k in (list(envs) if r % 2 == 0 else list(envs)[::-1]):
            ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            ev0.record()
            run(k, args.steps)
            ev1.record()
            torch.cuda.synchronize()
            ms[k].append(ev0.elapsed_time(ev1) / args.steps)
        o0, o1 = envs["no_bank"].observe(), envs["bank"].observe()
        same = same and all(torch.equal(a, b) for a, b in ((o0[0], o1[0]), (o0[1]["rgb"], o1[1]["rgb"]), (o0[2], o1[2])))
    ngames = len(game.split(","))
    out = {"config": f"{game if ngames == 1 else f'{ngames}-game list'} {mode} x{n} num_levels={levels}", "card": info,
           "steps_per_window": args.steps, "ms_per_step": ms,
           "env_steps_per_s": {k: [n / (v / 1e3) for v in ms[k]] for k in envs},
           "bank_build_s": build_s, "bank_levels": bank["levels"], "bank_bytes": bank["bytes"],
           "bank_bytes_per_level": bank["bytes"] / max(1, bank["levels"] * ngames),
           "outputs_equal": bool(same), "errors": {k: envs[k].errors() for k in envs}}
    print(json.dumps(out), flush=True)
    for e in envs.values():
        e.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200, help="steps per timed window")
    ap.add_argument("--rounds", type=int, default=3, help="timed windows per handle, alternating")
    ap.add_argument("--warmup", type=int, default=300, help="steps before the first window (spreads episode ends)")
    ap.add_argument("configs", nargs="*", default=DEFAULT)
    args = ap.parse_args()

    import torch

    from procgen_b200 import ProcgenGym3Env

    if not torch.cuda.is_available():
        raise SystemExit("level_bank_bench needs a CUDA device")
    torch.cuda.set_device(0)
    info = card()
    for cfg in args.configs:
        game, mode, n, levels = cfg.split(":")
        bench(torch, ProcgenGym3Env, game, mode, int(n), int(levels), args, info)


if __name__ == "__main__":
    main()
