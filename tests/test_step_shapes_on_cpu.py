"""Every combination of the six opt-ins of a step, in the host debug build: kernel launches and outputs.

pgb200_kernel_launches counts what a step issues, and the host debug build counts the loops that stand for the kernels
(step_shapes.expected_launches). test_outputs_per_step_shape also checks what the steps compute: step_shapes'
lockstep driver runs every shape of one game, and the 8 semantic shapes (level choice x pause x final outputs) with the
level bank, level lookahead and the rollout on for the 16-game list in 80 launches and the whole-world view, against
the oracle (its records, tests/golden/step_shape_records.json.gz; the live oracle while recording them). Every output,
final output, override entry, rollout slot and state blob is compared, and the launch count of every step. The GPU
build runs the same driver on the same records in tests/test_gpu_step_shapes.py."""
import pytest

from final_obs_oracle import LibFinal
from level_bank import build_bank
from level_lookahead import enable_lookahead
from level_seed_oracle import next_level_seeds
from oracle.ref_env import RefVecEnv, default_pack, mt19937_actions
from pause_oracle import pause_mask
from rollout import get_rollout
from step_shapes import (ALL_ON, MID_RUN_ORDERS, SHAPES, expected_launches, kernel_launches, mid_run_turn_on, run_case, semantic_shapes,
                         shape_id, use_step_shape_records)

KW = dict(distribution_mode="easy", num_levels=0, start_level=0, rand_seed=0)
# (env name, envs, launch_shape): one game in one launch, and a two-game list cut into 3 chunks per game
HANDLES = {"one_game": ("coinrun", 8, None), "two_games_3_chunks": ("coinrun,maze", 12, (3, False))}


@pytest.fixture(autouse=True, scope="module")
def _step_shape_records():
    use_step_shape_records()


@pytest.mark.parametrize("shape", SHAPES, ids=shape_id)
@pytest.mark.parametrize("handle", list(HANDLES))
def test_launches_per_step(hostsim_lib, handle, shape):
    name, n, launch_shape = HANDLES[handle]
    env = RefVecEnv(n, name, lib_path=hostsim_lib, resource_root=default_pack(), launch_shape=launch_shape, **KW)
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
        before = kernel_launches(env)
        env.act(a)
        assert kernel_launches(env) - before == expected_launches(shape, launches_per_step), f"step {t}"
    env.close()


# all 64 shapes of one game; the 8 semantic shapes with bank, lookahead and rollout on for the other cases
OUTPUT_RUNS = [("one_game", s) for s in SHAPES] + [(c, s) for c in ("sixteen_games", "whole_world") for s in semantic_shapes()]


@pytest.mark.parametrize("case,shape", OUTPUT_RUNS, ids=[f"{c}-{shape_id(s)}" for c, s in OUTPUT_RUNS])
def test_outputs_per_step_shape(hostsim_lib, case, shape):
    run_case(case, hostsim_lib, shape)


@pytest.mark.parametrize("order", list(MID_RUN_ORDERS))
def test_outputs_with_opt_ins_turned_on_mid_run(hostsim_lib, order):
    """One opt-in turned on every 4 steps, in three orders (the records test_gpu_step_shapes.py replays)"""
    run_case("sixteen_games", hostsim_lib, ALL_ON, turn_on=mid_run_turn_on(order), label=f"mid_run_{order}")
