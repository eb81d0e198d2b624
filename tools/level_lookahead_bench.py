"""What level lookahead (enable_level_lookahead) saves at num_levels = 0.

Per configuration, a handle without lookahead ("off") and one with it ("on"), same configuration. After a warm-up
that spreads episode ends, timed windows alternate between them; per window the device time per step (CUDA events on
the stepping stream) and env-steps/s. The outputs of the two handles are compared after every window: lookahead must not
change them. Then one window per handle under kernel timing: logic ms (logic and finish phase) and setup + render ms
per step, which shows where the time went. Also the counters (resets served from the slots, from a bank, generated)
and the bytes lookahead holds. One JSON line per configuration, with the card's name, power limit and maximum SM clock
read in the same process.

usage: python tools/level_lookahead_bench.py [--steps 200] [--rounds 3] [--warmup 300] [game:mode:envs ...]
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from tools.graph_step_bench import card  # noqa: E402

ALL16 = "bigfish,bossfight,caveflyer,chaser,climber,coinrun,dodgeball,fruitbot,heist,jumper,leaper,maze,miner,ninja,plunder,starpilot"
# coinrun easy at 65 536 is the headline configuration, where level generation is cheap: no gain is expected there
DEFAULT = [f"{g}:hard:32768" for g in ("caveflyer", "jumper", "leaper")] + [f"{ALL16}:hard:32768", "coinrun:easy:65536"]


def bench(torch, ProcgenGym3Env, game, mode, n, args, info):
    gen = torch.Generator(device="cuda").manual_seed(1234)
    T = 256
    actions = torch.randint(0, 15, (T, n), device="cuda", dtype=torch.int32, generator=gen)
    kw = dict(distribution_mode=mode, num_levels=0, start_level=0, rand_seed=0)
    envs = {"off": ProcgenGym3Env(n, game, **kw), "on": ProcgenGym3Env(n, game, **kw)}
    envs["on"].enable_level_lookahead()
    state = dict.fromkeys(envs, 0)

    def run(k, steps):
        for t in range(state[k], state[k] + steps):
            envs[k].act(actions[t % T])
        state[k] += steps

    for k in envs:
        run(k, args.warmup)
    torch.cuda.synchronize()
    counters0 = {k: envs[k].level_lookahead_info() for k in ("on",)}
    ms = {k: [] for k in envs}
    same = True
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
        o = {k: envs[k].observe() for k in envs}
        for k in ("on",):
            same = same and all(torch.equal(a, b) for a, b in ((o["off"][0], o[k][0]), (o["off"][1]["rgb"], o[k][1]["rgb"]),
                                                                (o["off"][2], o[k][2])))
            same = same and all(torch.equal(v, envs[k].get_info_tensors()[name]) for name, v in envs["off"].get_info_tensors().items())
    counters = {k: {c: v - counters0[k][c] if c != "bytes" else v for c, v in envs[k].level_lookahead_info().items()} for k in ("on",)}
    phases = {}
    steps_t = min(args.steps, 100)
    for k in envs:
        envs[k].kernel_timing_begin(steps_t * 128)
        run(k, steps_t)
        kt = envs[k].kernel_timing_end()
        phases[k] = {"logic_ms": kt["logic_ms"] / steps_t, "setup_plus_render_ms": (kt["setup_ms"] + kt["render_ms"]) / steps_t}
    ngames = len(game.split(","))
    out = {"config": f"{game if ngames == 1 else f'{ngames}-game list'} {mode} x{n} num_levels=0", "card": info,
           "steps_per_window": args.steps, "ms_per_step": ms,
           "env_steps_per_s": {k: [n / (v / 1e3) for v in ms[k]] for k in envs},
           "kernel_ms_per_step": phases, "lookahead": counters,
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
        raise SystemExit("level_lookahead_bench needs a CUDA device")
    torch.cuda.set_device(0)
    info = card()
    for cfg in args.configs:
        game, mode, n = cfg.split(":")
        bench(torch, ProcgenGym3Env, game, mode, int(n), args, info)


if __name__ == "__main__":
    main()
