"""Setup- and render-kernel phase cycles of one step (profiling variant libprocgen_b200_phase.so, -DPG_PHASE_TIMING).
usage: PROCGEN_B200_LIB=.../libprocgen_b200_phase.so python tools/gpu_render_phases.py game mode envs desync

SM cycles of each env's last frame, sampled over up to 512 envs. The two kernels write disjoint slots of the
header's 12 phase counters: the setup kernel 1-4, 8 and 9 (pg_kernels.cuh), the render kernel 0 and 5-7
(pg_launch.cuh). Cycles are per warp for the setup kernel and per CTA for the render kernel."""
import ctypes as C
import os
import struct
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from procgen_b200 import ProcgenGym3Env

KERNELS = {
    "setup": [(1, "setup_frame"), (2, "entity blits"), (3, "frame_build"), (4, "frame_tile_alloc"),
              (8, "frame_cells_finish"), (9, "record store")],
    "render": [(0, "stage (record + tiles)"), (5, "compose"), (6, "consumer + pack"), (7, "store")],
}

game, mode, n, desync = sys.argv[1], sys.argv[2], int(sys.argv[3]), int(sys.argv[4])
env = ProcgenGym3Env(n, game, distribution_mode=mode, num_levels=0, rand_seed=0)
off = env._lib.pgb200_debug_phase_offset()
assert off >= 0, "needs the PG_PHASE_TIMING build"
g = torch.Generator(device="cuda").manual_seed(0)
acts = torch.randint(0, 15, (64, n), device="cuda", dtype=torch.int32, generator=g)
for t in range(desync):
    env.act(acts[t % 64])
env.observe()
torch.cuda.synchronize()
buf = (C.c_ubyte * 1024)()
acc = []
for e in range(0, n, max(1, n // 512)):
    env._lib.pgb200_debug_read_env(env._h, int(e), buf, None, 0)
    acc.append(struct.unpack_from("<12I", bytes(buf), off))
a = np.array(acc, dtype=np.float64)
print(f"{game} {mode}, {n} envs, after {desync} steps ({len(a)} envs sampled)")
for kernel, phases in KERNELS.items():
    tot = sum(a[:, i].mean() for i, _ in phases)
    print(f"  {kernel} kernel: mean cycles per frame {tot:.0f}")
    for i, nm in phases:
        print(f"    [{i:2d}] {nm:22s} mean {a[:, i].mean():8.0f}  p90 {np.percentile(a[:, i], 90):8.0f}  {100 * a[:, i].mean() / tot:5.1f}%")
env.close()
