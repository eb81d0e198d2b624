"""Host cost of a device-resident step, eager next to a CUDA-graph replay of the same step.

For each configuration two device-resident handles of the same envs: `eager` calls act() every step, `graph`
captured one act() in a torch.cuda.CUDAGraph and replays it (the step's actions are copied into the graph's
action buffer first; act() does the same copy into the library's buffer). After a desynchronising rollout,
timed windows of the two alternate. Per window: the host µs per step (the host clock around the issue of the
steps, before the closing synchronise) and env-steps/s (CUDA events on the stepping stream around the window).
One JSON line per configuration, with the card's name, power limit and maximum SM clock read in the same
process.

usage: python tools/graph_step_bench.py [--steps 300] [--rounds 4] [--desync 300] [game:mode:envs ...]
(default configurations: coinrun:easy:64 coinrun:easy:4096 coinrun:easy:65536 and the 16-game list at 2048 envs
per game, "all16:hard:32768")
"""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

ALL16 = "bigfish,bossfight,caveflyer,chaser,climber,coinrun,dodgeball,fruitbot,heist,jumper,leaper,maze,miner,ninja,plunder,starpilot"


def card():
    import torch

    out = {"name": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        out["power_limit"], out["sm_max_clock"] = [x.strip() for x in q.split(",")]
    except Exception as e:  # noqa: BLE001 - the numbers are still reported, without the card's limits
        out["nvidia_smi"] = repr(e)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=300, help="steps per timed window")
    ap.add_argument("--rounds", type=int, default=4, help="timed windows per mode, alternating")
    ap.add_argument("--desync", type=int, default=300)
    ap.add_argument("configs", nargs="*", default=["coinrun:easy:64", "coinrun:easy:4096", "coinrun:easy:65536", "all16:hard:32768"])
    args = ap.parse_args()

    import torch

    from procgen_b200 import ProcgenGym3Env

    if not torch.cuda.is_available():
        raise SystemExit("graph_step_bench needs a CUDA device")
    torch.cuda.set_device(0)
    info = card()
    K = args.steps
    for cfg in args.configs:
        game, mode, n = cfg.split(":")
        n = int(n)
        name = ALL16 if game == "all16" else game
        gen = torch.Generator(device="cuda").manual_seed(1234)
        T = 256
        actions = torch.randint(0, 15, (T, n), device="cuda", dtype=torch.int32, generator=gen)
        envs = {k: ProcgenGym3Env(n, name, distribution_mode=mode, num_levels=0, start_level=0, rand_seed=0) for k in ("eager", "graph")}
        a = torch.zeros(n, dtype=torch.int32, device="cuda")
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            envs["graph"].act(a)
        state = {"eager": 0, "graph": 0}

        def run(k, steps):
            t0 = state[k]
            if k == "eager":
                env = envs["eager"]
                for t in range(t0, t0 + steps):
                    env.act(actions[t % T])
            else:
                for t in range(t0, t0 + steps):
                    a.copy_(actions[t % T])
                    g.replay()
            state[k] = t0 + steps

        for k in envs:
            run(k, args.desync)
        torch.cuda.synchronize()
        stats = {k: {"host_us": [], "ms": []} for k in envs}
        for r in range(args.rounds):
            for k in (("eager", "graph") if r % 2 == 0 else ("graph", "eager")):
                ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                torch.cuda.synchronize()
                ev0.record()
                h0 = time.perf_counter()
                run(k, K)
                h1 = time.perf_counter()
                ev1.record()
                torch.cuda.synchronize()
                stats[k]["host_us"].append((h1 - h0) * 1e6 / K)
                stats[k]["ms"].append(ev0.elapsed_time(ev1))
        rate = {k: [K * n / (ms / 1e3) for ms in stats[k]["ms"]] for k in envs}
        out = {
            "config": f"{game} {mode} x{n}", "card": info, "steps_per_window": K, "rounds": args.rounds,
            "host_us_per_step": {k: stats[k]["host_us"] for k in envs},
            "env_steps_per_s": rate,
            "graph_over_eager_best_rate": max(rate["graph"]) / max(rate["eager"]),
            "errors": {k: envs[k].errors() for k in envs},
        }
        print(json.dumps(out), flush=True)
        for env in envs.values():
            env.close()


if __name__ == "__main__":
    main()
