"""Steady-state env-steps/s with per-env level-seed overrides in use, next to the same loop without them.

Two device-resident handles of the same configuration: `plain` never requests the override array (the
library's default path), `override` has every consumed entry refilled by torch before every step (one
elementwise kernel on the stepping stream, part of what a caller pays), so every episode end plays a
caller-chosen level. After a desynchronising rollout (episode ends spread over the steps), timed windows of
the two alternate (CUDA events on the stepping stream). One JSON line per configuration, with the card's name,
power limit and maximum SM clock read in the same process.

usage: python tools/level_seed_bench.py [--envs 65536] [--steps 200] [--rounds 3] [--desync 1000] [game:mode ...]
(default configurations: coinrun:easy bigfish:hard)
"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


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
    ap.add_argument("--envs", type=int, default=65536)
    ap.add_argument("--steps", type=int, default=200, help="steps per timed window")
    ap.add_argument("--rounds", type=int, default=3, help="timed windows per handle, alternating")
    ap.add_argument("--desync", type=int, default=1000)
    ap.add_argument("configs", nargs="*", default=["coinrun:easy", "bigfish:hard"])
    args = ap.parse_args()

    import torch

    from procgen_b200 import ProcgenGym3Env

    if not torch.cuda.is_available():
        raise SystemExit("level_seed_bench needs a CUDA device")
    torch.cuda.set_device(0)
    info = card()
    n, K = args.envs, args.steps
    for cfg in args.configs:
        game, mode = cfg.split(":")
        gen = torch.Generator(device="cuda").manual_seed(1234)
        T = 256
        actions = torch.randint(0, 15, (T, n), device="cuda", dtype=torch.int32, generator=gen)
        pool = torch.randint(0, 2 ** 31 - 1, (8, n), device="cuda", dtype=torch.int32, generator=gen)
        envs = {k: ProcgenGym3Env(n, game, distribution_mode=mode, num_levels=0, start_level=0, rand_seed=0) for k in ("plain", "override")}
        seeds = envs["override"].next_level_seeds()
        state = {"plain": 0, "override": 0}   # steps taken by each handle (actions index)
        stats = {k: {"ms": [], "first": 0, "taken": 0} for k in envs}

        def run(k, steps, count=False):
            env = envs[k]
            t0 = state[k]
            firsts = torch.zeros((), device="cuda", dtype=torch.int64)
            taken = torch.zeros((), device="cuda", dtype=torch.int64)
            for t in range(t0, t0 + steps):
                if k == "override":
                    seeds.copy_(torch.where(seeds < 0, pool[t % 8], seeds))
                    if count:
                        pend = seeds >= 0
                env.act(actions[t % T])
                rew, ob, first = env.observe()
                if count:
                    firsts += first.sum()
                    if k == "override":
                        taken += (pend & (seeds < 0)).sum()
            state[k] = t0 + steps
            return int(firsts.item()), int(taken.item())

        for k in envs:
            run(k, args.desync)
        torch.cuda.synchronize()
        for r in range(args.rounds):
            for k in (("plain", "override") if r % 2 == 0 else ("override", "plain")):
                ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                torch.cuda.synchronize()
                ev0.record()
                run(k, K)
                ev1.record()
                torch.cuda.synchronize()
                stats[k]["ms"].append(ev0.elapsed_time(ev1))
        # an untimed pass of the same length: how many env-steps end an episode, how many take an override
        for k in envs:
            stats[k]["first"], stats[k]["taken"] = run(k, K, count=True)
        rate = {k: [K * n / (ms / 1e3) for ms in stats[k]["ms"]] for k in envs}
        best = {k: max(v) for k, v in rate.items()}
        out = {
            "config": f"{game} {mode} x{n}", "card": info, "steps_per_window": K, "rounds": args.rounds,
            "plain_env_steps_per_s": rate["plain"], "override_env_steps_per_s": rate["override"],
            "override_over_plain_best": best["override"] / best["plain"],
            "episode_ends_per_env_step": {k: stats[k]["first"] / (K * n) for k in envs},
            "overrides_taken_per_env_step": stats["override"]["taken"] / (K * n),
            "errors": {k: envs[k].errors() for k in envs},
        }
        print(json.dumps(out), flush=True)
        for env in envs.values():
            env.close()


if __name__ == "__main__":
    main()
