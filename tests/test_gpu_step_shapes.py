"""Every combination of the six opt-ins of a step on the GPU, against the oracle's records.

A step's kernels come from its shape: level choice, pause mask, final outputs, level bank, level lookahead and rollout
(StepShape, pg_launch.cuh), and each phase turns the flags it depends on into template arguments. The host debug build
never compiles the device-only paths those instantiations take (warp-wide list appends, lane-0 slot keying in
lookahead_predict, the atomic counters, the lookahead side stream, the fixed grids of phase B's frames), so the matrix
runs here as well: step_shapes.run_shape_lockstep against tests/golden/step_shape_records.json.gz, which the host
debug build's test_step_shapes_on_cpu.py recorded against the live oracle. Then the opt-ins turned on one by one in a
handle that is already stepping, and an 8-step CUDA graph with all of them and the fp16 consumer output against eager
steps of an identical handle."""
import pytest

from oracle.record import STANDIN_PACK
from step_shapes import (ALL16, ALL_ON, BANK_SEEDS, CASES, MID_RUN_ORDERS, OVERRIDE_SEEDS, case_shapes, mid_run_turn_on,
                         run_case, shape_id, use_step_shape_records)

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True, scope="module")
def _step_shape_records():
    use_step_shape_records()


MATRIX = [(case, shape, ls) for case in CASES for shape, ls in case_shapes(case)]


def _run_id(case, shape, ls):
    return f"{case}-{shape_id(shape)}" + ("-serialized" if ls and ls[1] else "")


@pytest.mark.parametrize("case,shape,launch_shape", MATRIX, ids=[_run_id(*m) for m in MATRIX])
def test_step_shape_against_record(product_lib, case, shape, launch_shape):
    run_case(case, product_lib, shape, launch_shape)


@pytest.mark.parametrize("order", list(MID_RUN_ORDERS))
def test_opt_ins_turned_on_mid_run(product_lib, order):
    """One opt-in every 4 steps on the 16-game list in 80 launches: lookahead's bulk fill, the rollout's slot 0 and the
    first final outputs of a handle that is already stepping."""
    run_case("sixteen_games", product_lib, ALL_ON, turn_on=mid_run_turn_on(order), label=f"mid_run_{order}")


def test_captured_step_with_everything_on(product_lib):
    """4 096 envs of the 16-game list in 80 launches with all six opt-ins and the fp16 consumer output (k = 4): an 8-step
    graph in which torch refills the consumed overrides (half of them, from a pool over [0, 400)) and the pause mask
    before every act(), replayed 6 times, equals eager steps of an identical handle with the same writes: outputs, final
    outputs, rollout, override array, consumer ring, lookahead counters after every replay, state blobs at the end. The
    rollout has 8 slots, so that it holds rew, rgb and first of every step of a replay."""
    import torch

    from procgen_b200 import ProcgenGym3Env

    n, k, reps = 4096, 4, 6
    kw = dict(distribution_mode="hard", num_levels=0, start_level=0, rand_seed=0, resource_root=STANDIN_PACK)
    envs = [ProcgenGym3Env(n, ALL16, **kw) for _ in range(2)]
    views = []
    for env in envs:
        env.set_launch_shape(5)
        v = {"seeds": env.next_level_seeds(), "mask": env.pause_mask(), "final": env.final_outputs(), "roll": env.rollout(8)}
        env.build_level_bank(BANK_SEEDS)
        env.enable_level_lookahead()
        env.enable_consumer_output(torch.float16, frames=k)
        v["slot"], v["ring"] = env.consumer_slot_tensor(), env.consumer_ring()
        views.append(v)
    gen = torch.Generator(device="cuda").manual_seed(12)
    total = 2 + reps * 8
    acts = torch.randint(0, 15, (total, n), device="cuda", dtype=torch.int32, generator=gen)
    acts[torch.rand((total, n), device="cuda", generator=gen) < 1 / 6] = -1
    masks = (torch.rand((total, n), device="cuda", generator=gen) < 0.5).to(torch.uint8)
    pools = torch.randint(*OVERRIDE_SEEDS, (total, n), device="cuda", dtype=torch.int32, generator=gen)
    refill = torch.rand((total, n), device="cuda", generator=gen) < 0.5

    def step(env, v, a, m, pool, sel):
        v["seeds"].copy_(torch.where(sel & (v["seeds"] < 0), pool, v["seeds"]))
        v["mask"].copy_(m)
        env.act(a)

    # two eager steps on both handles first: every kernel of the shape has run once before the capture
    for t in range(2):
        for env, v in zip(envs, views):
            step(env, v, acts[t], masks[t], pools[t], refill[t])
    graph, eager = envs
    gv, ev = views
    bufs = [torch.zeros((8, n), device="cuda", dtype=x.dtype) for x in (acts, masks, pools, refill)]
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for s in range(8):
            step(graph, gv, *(b[s] for b in bufs))
    ended = 0
    for r in range(reps):
        sl = slice(2 + 8 * r, 10 + 8 * r)
        for b, x in zip(bufs, (acts, masks, pools, refill)):
            b.copy_(x[sl])
        g.replay()
        for t in range(sl.start, sl.stop):
            step(eager, ev, acts[t], masks[t], pools[t], refill[t])
        torch.cuda.synchronize()
        for what, a, b in [("rew", graph.observe()[0], eager.observe()[0]), ("rgb", graph.observe()[1]["rgb"], eager.observe()[1]["rgb"]),
                           ("first", graph.observe()[2], eager.observe()[2])] + \
                [(f"info {key}", graph.get_info_tensors()[key], eager.get_info_tensors()[key]) for key in graph.get_info_tensors()] + \
                [(f"final {key}", gv["final"][key], ev["final"][key]) for key in gv["final"]] + \
                [(f"rollout {key}", gv["roll"][key], ev["roll"][key]) for key in gv["roll"]] + \
                [(key, gv[key], ev[key]) for key in ("seeds", "mask", "slot", "ring")]:
            assert torch.equal(a, b), f"replay {r}: {what} differs"
        ended += int((ev["final"]["level_end"] != 0).sum())
        assert graph.level_lookahead_info() == eager.level_lookahead_info(), f"replay {r}: lookahead counters"
    info = eager.level_lookahead_info()
    assert ended > 0 and info["served"] > 0 and info["bank"] > 0 and info["generated"] > 0, info
    assert graph.get_state() == eager.get_state(), "state blobs differ at the end"
    assert graph.errors() == 0 and eager.errors() == 0
    for env in envs:
        env.close()
