"""What action repeat (pgb200_get_action_repeat) costs against the same game steps taken from outside.

Per configuration and repeat count r in --repeats: one handle with every count set to r, whose act() plays up to r game
steps and renders once, and one handle without counts that takes r plain steps per act() and throws r - 1 frames away
(what a caller does without the feature, apart from the pause mask it would also need to stop at an episode's end).
After a desynchronising rollout, timed windows alternate between the two; per window the device time per act() (CUDA
events on the stepping stream), and the ratio of the two handles' best windows. The repeat handle may play fewer game
steps than r where an episode ends inside an act(), so the ratio is the saving per act(), not per game step.
One JSON line per measurement, with the card's name, power limit and maximum SM clock read in the same process.

usage: python tools/action_repeat_bench.py [--steps 100] [--rounds 3] [--desync 200] [--repeats 1,2,4,8] [game:mode:envs ...]
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from tools.graph_step_bench import card  # noqa: E402

ALL16 = "bigfish,bossfight,caveflyer,chaser,climber,coinrun,dodgeball,fruitbot,heist,jumper,leaper,maze,miner,ninja,plunder,starpilot"


def act_time(torch, ProcgenGym3Env, game, mode, n, r, args, info):
    gen = torch.Generator(device="cuda").manual_seed(1234)
    T = 256
    actions = torch.randint(0, 15, (T, n), device="cuda", dtype=torch.int32, generator=gen)
    kw = dict(distribution_mode=mode, num_levels=0, start_level=0, rand_seed=0)
    envs = {"repeat": ProcgenGym3Env(n, game, **kw), "plain_steps": ProcgenGym3Env(n, game, **kw)}
    state = dict.fromkeys(envs, 0)

    def run(k, acts):
        for t in range(state[k], state[k] + acts):
            for _ in range(1 if k == "repeat" else r):
                envs[k].act(actions[t % T])
        state[k] += acts

    for k in envs:  # the desynchronising rollout runs one game step per act() on both
        for t in range(args.desync):
            envs[k].act(actions[t % T])
    envs["repeat"].action_repeat().fill_(r)
    for k in envs:
        run(k, 2)
    torch.cuda.synchronize()
    ms = {k: [] for k in envs}
    kinds = list(envs)
    for i in range(args.rounds):
        for k in (kinds if i % 2 == 0 else kinds[::-1]):
            ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            ev0.record()
            run(k, args.steps)
            ev1.record()
            torch.cuda.synchronize()
            ms[k].append(ev0.elapsed_time(ev1) / args.steps)
    out = {"measure": "act_time", "config": f"{game if game != ALL16 else '16-game list'} {mode} x{n}", "repeat": r,
           "card": info, "acts_per_window": args.steps, "ms_per_act": ms,
           "speedup": min(ms["plain_steps"]) / min(ms["repeat"]), "errors": {k: e.errors() for k, e in envs.items()}}
    print(json.dumps(out), flush=True)
    for e in envs.values():
        e.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=100, help="act() calls per timed window")
    ap.add_argument("--rounds", type=int, default=3, help="timed windows per handle, alternating")
    ap.add_argument("--desync", type=int, default=200)
    ap.add_argument("--repeats", default="1,2,4,8")
    ap.add_argument("configs", nargs="*", default=["coinrun:easy:65536", "all16:hard:65536"])
    args = ap.parse_args()

    import torch

    from procgen_b200 import ProcgenGym3Env

    if not torch.cuda.is_available():
        raise SystemExit("action_repeat_bench needs a CUDA device")
    torch.cuda.set_device(0)
    info = card()
    for cfg in args.configs:
        game, mode, n = cfg.split(":")
        for r in (int(x) for x in args.repeats.split(",")):
            act_time(torch, ProcgenGym3Env, ALL16 if game == "all16" else game, mode, int(n), r, args, info)


if __name__ == "__main__":
    main()
