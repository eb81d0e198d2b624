"""Cost of final outputs (pgb200_get_final_outputs), and how often levels end per cause.

For each configuration four device-resident handles of the same envs: with and without final outputs, each stepped
eagerly (act() every step) and by replaying a CUDA graph of one act(). After a desynchronising rollout, timed
windows of the four alternate. Per window: the host µs per step (the host clock around the issue of the steps,
before the closing synchronise) and env-steps/s (CUDA events on the stepping stream around the window). Then an
untimed run of the eager final-outputs handle counts level_end per game and cause: how often a level ends by the
game (death or completion), by the time limit (a truncation) or by the caller (action -1, never here: actions are
uniform over 0..14). One JSON line per configuration, with the card's name, power limit and maximum SM clock read in
the same process.

usage: python tools/final_obs_bench.py [--steps 300] [--rounds 4] [--desync 300] [--mix-steps 2000] [game:mode:envs ...]
(default configurations: coinrun:easy:65536 bigfish:hard:65536 all16:hard:32768, the 16-game list at 2048 envs per game)
"""
import argparse
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from tools.graph_step_bench import ALL16, card  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=300, help="steps per timed window")
    ap.add_argument("--rounds", type=int, default=4, help="timed windows per handle, alternating")
    ap.add_argument("--desync", type=int, default=300)
    ap.add_argument("--mix-steps", type=int, default=2000, help="steps of the level-end count")
    ap.add_argument("configs", nargs="*", default=["coinrun:easy:65536", "bigfish:hard:65536", "all16:hard:32768"])
    args = ap.parse_args()

    import torch

    from procgen_b200 import ProcgenGym3Env

    if not torch.cuda.is_available():
        raise SystemExit("final_obs_bench needs a CUDA device")
    torch.cuda.set_device(0)
    info = card()
    K = args.steps
    kinds = ("eager", "eager_final", "graph", "graph_final")
    for cfg in args.configs:
        game, mode, n = cfg.split(":")
        n = int(n)
        name = ALL16 if game == "all16" else game
        games = name.split(",")
        gen = torch.Generator(device="cuda").manual_seed(1234)
        T = 256
        actions = torch.randint(0, 15, (T, n), device="cuda", dtype=torch.int32, generator=gen)
        envs = {k: ProcgenGym3Env(n, name, distribution_mode=mode, num_levels=0, start_level=0, rand_seed=0) for k in kinds}
        for k in ("eager_final", "graph_final"):
            envs[k].final_outputs()
        graphs, acts = {}, {}
        for k in ("graph", "graph_final"):
            acts[k] = torch.zeros(n, dtype=torch.int32, device="cuda")
            graphs[k] = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graphs[k]):
                envs[k].act(acts[k])
        state = dict.fromkeys(kinds, 0)

        def run(k, steps):
            t0 = state[k]
            for t in range(t0, t0 + steps):
                if k in graphs:
                    acts[k].copy_(actions[t % T])
                    graphs[k].replay()
                else:
                    envs[k].act(actions[t % T])
            state[k] = t0 + steps

        for k in kinds:
            run(k, args.desync)
        torch.cuda.synchronize()
        stats = {k: {"host_us": [], "ms": []} for k in kinds}
        for r in range(args.rounds):
            for k in (kinds if r % 2 == 0 else kinds[::-1]):
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
        rate = {k: [K * n / (ms / 1e3) for ms in stats[k]["ms"]] for k in kinds}
        # level-end mix: env e plays games[e % G]
        env = envs["eager_final"]
        level_end = env.final_outputs()["level_end"]
        game_of = torch.arange(n, device="cuda") % len(games)
        counts = torch.zeros(len(games) * 4, dtype=torch.int64, device="cuda")
        for t in range(args.mix_steps):
            env.act(actions[t % T])
            counts += torch.bincount(game_of * 4 + level_end.long(), minlength=len(games) * 4)
        counts = counts.view(len(games), 4).cpu().tolist()
        env_steps = args.mix_steps * n // len(games)
        mix = {g: {"env_steps": env_steps, "game": c[1], "timeout": c[2], "caller": c[3],
                   "ends_per_env_step_pct": round(100.0 * (c[1] + c[2] + c[3]) / env_steps, 3),
                   "timeout_share_of_ends_pct": round(100.0 * c[2] / max(1, c[1] + c[2] + c[3]), 2)} for g, c in zip(games, counts)}
        out = {
            "config": f"{game} {mode} x{n}", "card": info, "steps_per_window": K, "rounds": args.rounds,
            "host_us_per_step": {k: stats[k]["host_us"] for k in kinds},
            "env_steps_per_s": rate,
            "final_over_plain_best_rate": {"eager": max(rate["eager_final"]) / max(rate["eager"]),
                                           "graph": max(rate["graph_final"]) / max(rate["graph"])},
            "level_end_mix": mix,
            "errors": {k: envs[k].errors() for k in kinds},
        }
        print(json.dumps(out), flush=True)
        for e in envs.values():
            e.close()


if __name__ == "__main__":
    main()
