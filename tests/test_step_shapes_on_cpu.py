"""Kernel launches per step for every combination of the six opt-ins, in the host debug build.

pgb200_kernel_launches counts what a step issues, and the host debug build counts the loops that stand for the kernels.
Per (game, env chunk) launch, a plain step issues 3: logic, setup and render. A two-phase step without final outputs (a
level bank or level lookahead) issues 4, with the finish kernel. A step with final outputs issues 6: it renders in both
phases. Level lookahead adds its own kernel. The rollout adds one per step, the advance of its cursor. The level-seed
overrides and the pause mask select other instantiations of the same kernels and add none."""
import ctypes as C
import itertools

import pytest

from final_obs_oracle import LibFinal
from level_bank import build_bank
from level_lookahead import enable_lookahead
from level_seed_oracle import next_level_seeds
from oracle.ref_env import RefVecEnv, default_pack, mt19937_actions
from pause_oracle import pause_mask
from rollout import get_rollout

OPT_INS = ("level_choice", "pause", "final", "bank", "look", "roll")
SHAPES = [dict(zip(OPT_INS, bits)) for bits in itertools.product((False, True), repeat=len(OPT_INS))]
KW = dict(distribution_mode="easy", num_levels=0, start_level=0, rand_seed=0)
# (env name, envs, launch_shape): one game in one launch, and a two-game list cut into 3 chunks per game
HANDLES = {"one_game": ("coinrun", 8, None), "two_games_3_chunks": ("coinrun,maze", 12, (3, False))}


def _shape_id(shape):
    return "+".join(k for k in OPT_INS if shape[k]) or "plain"


def expected_launches(shape, launches_per_step):
    if shape["final"]:
        per_launch = 6
    elif shape["bank"] or shape["look"]:
        per_launch = 4
    else:
        per_launch = 3
    if shape["look"]:
        per_launch += 1
    return per_launch * launches_per_step + (1 if shape["roll"] else 0)


@pytest.mark.parametrize("shape", SHAPES, ids=_shape_id)
@pytest.mark.parametrize("handle", list(HANDLES))
def test_launches_per_step(hostsim_lib, handle, shape):
    name, n, launch_shape = HANDLES[handle]
    env = RefVecEnv(n, name, lib_path=hostsim_lib, resource_root=default_pack(), launch_shape=launch_shape, **KW)
    lib = env.lib
    lib.pgb200_kernel_launches.argtypes = [C.c_void_p]
    lib.pgb200_kernel_launches.restype = C.c_int64
    if shape["level_choice"]:
        next_level_seeds(env)
    if shape["pause"]:
        mask = pause_mask(env)
        mask[::2] = 1  # half the envs held still: a paused env changes what a launch does, not what it issues
    if shape["final"]:
        LibFinal(env)
    if shape["bank"]:
        assert build_bank(env, [1, 2, 3], capacity=4) == 0
    if shape["look"]:
        assert enable_lookahead(env) == 0
    if shape["roll"]:
        assert get_rollout(env, 3)[0] == 0
    games = len(name.split(","))
    launches_per_step = games * (launch_shape[0] if launch_shape else 1)
    for t, a in enumerate(mt19937_actions(3, n, 4)):
        before = lib.pgb200_kernel_launches(C.c_void_p(env.h))
        env.act(a)
        assert lib.pgb200_kernel_launches(C.c_void_p(env.h)) - before == expected_launches(shape, launches_per_step), f"step {t}"
    env.close()
