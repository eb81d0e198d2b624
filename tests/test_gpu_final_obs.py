"""Final outputs (pgb200_get_final_outputs) on the GPU.

The cases of test_final_obs_on_cpu.py against the oracle's records (tests/golden/final_obs_records.json.gz, in which
level_end and the final frames are folded with the outputs; recorded with the final-frame hook on the oracle), and at benchmark
size through the device-resident Python API: 65 536 envs (8 launch chunks per game) whose every output, consumer
ring included, equals an untouched control handle's, 64 of them followed by the oracle with their final frames. Also
a CUDA graph of 8 steps equal to eager stepping, and the Python accessor's rules."""
import ctypes as C

import numpy as np
import pytest

from final_obs_oracle import final_oracle_env, force_plan, near_timeout, run_final_lockstep, use_final_obs_records
from level_seed_oracle import refill_plan
from oracle.record import STANDIN_PACK
from oracle.ref_env import MAX_STATE_SIZE, RefVecEnv

pytestmark = pytest.mark.gpu

ALL16 = "bigfish,bossfight,caveflyer,chaser,climber,coinrun,dodgeball,fruitbot,heist,jumper,leaper,maze,miner,ninja,plunder,starpilot"
KW = dict(distribution_mode="hard", num_levels=200, start_level=0, rand_seed=0)


@pytest.fixture(autouse=True, scope="module")
def _final_obs_records():
    use_final_obs_records()


def _pair(lib, n, name, launch_shape=None, **kw):
    ref, fin = final_oracle_env(n, name, lib, **kw)
    dut = RefVecEnv(n, name, lib_path=lib, resource_root=STANDIN_PACK, launch_shape=launch_shape, **kw)
    return ref, fin, dut


def _close(*envs):
    for e in envs:
        e.close()


def test_sixteen_games_game_and_caller_ends(product_lib):
    ref, fin, dut = _pair(product_lib, 16, ALL16, **KW)
    ends = run_final_lockstep(ref, fin, dut, 300, plan=force_plan(1))
    assert (ends == 1).any() and (ends == 3).any()
    _close(ref, fin, dut)


def test_timeout_in_every_game(product_lib):
    n = 32
    ref, fin, dut = _pair(product_lib, n, ALL16, **KW)
    near_timeout([ref, dut], n)
    ends = run_final_lockstep(ref, fin, dut, 40)
    assert {e % 16 for e in np.nonzero((ends == 2).any(0))[0]} == set(range(16))
    _close(ref, fin, dut)


def test_sequential_levels(product_lib):
    kw = dict(distribution_mode="easy", num_levels=3, start_level=0, rand_seed=0, use_sequential_levels=True)
    ref, fin, dut = _pair(product_lib, 8, "maze", **kw)
    assert (run_final_lockstep(ref, fin, dut, 300, sequential=True) == 1).any()
    _close(ref, fin, dut)


@pytest.mark.parametrize("name", ["coinrun", "climber", "caveflyer", "ninja", "jumper"])
def test_whole_world_view(product_lib, name):
    ref, fin, dut = _pair(product_lib, 8, name, **dict(KW, center_agent=False))
    assert run_final_lockstep(ref, fin, dut, 150, plan=force_plan(2, every=8)).any()
    _close(ref, fin, dut)


def test_overrides_refilled_every_step(product_lib):
    ref, fin, dut = _pair(product_lib, 32, ALL16, **KW)
    assert (run_final_lockstep(ref, fin, dut, 200, plan=refill_plan(32, 1), overrides=True) == 3).any()
    _close(ref, fin, dut)


@pytest.mark.parametrize("chunks", [3, 64])
def test_forced_launch_shapes(product_lib, chunks):
    n = 48 if chunks == 3 else 32
    ref, fin, dut = _pair(product_lib, n, ALL16, launch_shape=(chunks, False), **KW)
    assert run_final_lockstep(ref, fin, dut, 150, plan=force_plan(3)).any()
    _close(ref, fin, dut)


# ------------------------------------------------------------------ benchmark size, device-resident
@pytest.mark.parametrize("name,mode", [("coinrun", "easy"), ("bigfish,coinrun", "hard")])
def test_final_outputs_at_size(product_lib, name, mode):
    """65 536 envs, one action in 16 set to -1, the consumer output on (k = 4). Every step every output of the
    handle with final outputs, its consumer ring included, equals a control handle's without them, level_end != 0
    exactly where first is set, and 64 envs from all over the array, exported into a 64-env oracle, have the
    oracle's level_end and final frames."""
    import torch

    from procgen_b200 import ProcgenGym3Env

    n_big, n_pick, warm, steps, k = 65536, 64, 20, 200, 4
    n_games = len(name.split(","))
    rs = np.random.RandomState(17)
    picks = []
    for j in range(n_pick):   # pick j plays game j % n_games, one pick per 1/64 of the array
        lo, hi = j * (n_big // n_pick), (j + 1) * (n_big // n_pick)
        e = int(rs.randint(lo, hi))
        e = e - (e % n_games) + (j % n_games)
        if e >= hi:
            e -= n_games
        picks.append(e)
    picks = np.array(picks)
    pick_t = torch.as_tensor(picks, device="cuda")
    kw = dict(distribution_mode=mode, num_levels=0, start_level=0, rand_seed=0, resource_root=STANDIN_PACK)
    env = ProcgenGym3Env(n_big, name, **kw)
    ctl = ProcgenGym3Env(n_big, name, **kw)
    for h in (env, ctl):
        h.enable_consumer_output(dtype=torch.float16, frames=k)
    final = env.final_outputs()
    assert not bool(final["level_end"].any()) and not bool(final["rgb"].any())
    gen = torch.Generator(device="cuda").manual_seed(21)
    acts = torch.randint(0, 15, (warm + steps, n_big), device="cuda", dtype=torch.int32, generator=gen)
    acts[torch.rand((warm + steps, n_big), device="cuda", generator=gen) < 1 / 16] = -1
    for t in range(warm):
        env.act(acts[t])
        ctl.act(acts[t])
    env.observe()
    buf = C.create_string_buffer(MAX_STATE_SIZE)

    def blob(e):
        nbytes = int(env._lib.get_state(env._h, int(e), buf, MAX_STATE_SIZE))
        return bytes(buf.raw[:nbytes])

    ref, fin = final_oracle_env(n_pick, name, product_lib, distribution_mode=mode, num_levels=0, start_level=0, rand_seed=99)
    for j, e in enumerate(picks):
        ref.set_state(j, blob(e))
    ref.observe()
    ends = 0
    for t in range(warm, warm + steps):
        a = acts[t][pick_t].cpu().numpy()
        fin.prepare(a)
        ref.act(a)
        env.act(acts[t])
        ctl.act(acts[t])
        rew, ob, first = env.observe()
        crew, cob, cfirst = ctl.observe()
        assert torch.equal(ob["rgb"], cob["rgb"]) and torch.equal(rew, crew) and torch.equal(first, cfirst), f"step {t}"
        for key, v in env.get_info_tensors().items():
            assert torch.equal(v, ctl.get_info_tensors()[key]), f"step {t}: info {key}"
        assert torch.equal(env.consumer_ring(), ctl.consumer_ring()), f"step {t}: consumer ring"
        le = final["level_end"]
        assert torch.equal(le != 0, first), f"step {t}: level_end against first"
        r, o, f = ref.observe()
        le_r, rgb_r = fin.read()
        ref._fold(le_r, rgb_r[le_r != 0])
        assert np.array_equal(rew[pick_t].cpu().numpy(), r) and np.array_equal(o["rgb"], ob["rgb"][pick_t].cpu().numpy()), f"step {t}"
        assert np.array_equal(le[pick_t].cpu().numpy(), le_r), f"step {t}: level_end of the followed envs"
        ended = le_r != 0
        assert np.array_equal(final["rgb"][pick_t].cpu().numpy()[ended], rgb_r[ended]), f"step {t}: final frames of the followed envs"
        ends += int((le != 0).sum())
    for j, e in enumerate(picks):
        assert blob(e) == ref.get_state(j), f"state blob of env {e} at the end"
    assert ends > n_big // 8
    assert env.errors() == 0 and ctl.errors() == 0
    for h in (env, ctl, ref, fin):
        h.close()


# ------------------------------------------------------------------ CUDA graphs, Python API
def test_graph_of_eight_steps_equals_eager(product_lib):
    """A graph of 8 act() calls with final outputs on, replayed, computes what eager steps compute: outputs,
    level_end and final frames after every replay."""
    import torch

    from procgen_b200 import ProcgenGym3Env

    n, reps = 4096, 12
    kw = dict(distribution_mode="hard", num_levels=0, start_level=0, rand_seed=5, resource_root=STANDIN_PACK)
    ALL2 = "bigfish,coinrun"
    eager = ProcgenGym3Env(n, ALL2, **kw)
    graph = ProcgenGym3Env(n, ALL2, **kw)
    fe, fg = eager.final_outputs(), graph.final_outputs()
    gen = torch.Generator(device="cuda").manual_seed(4)
    acts = torch.randint(0, 15, (reps * 8, n), device="cuda", dtype=torch.int32, generator=gen)
    acts[torch.rand((reps * 8, n), device="cuda", generator=gen) < 1 / 16] = -1
    buf = torch.zeros((8, n), device="cuda", dtype=torch.int32)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for s in range(8):
            graph.act(buf[s])
    torch.cuda.synchronize()
    ends = 0
    for r in range(reps):
        buf.copy_(acts[8 * r:8 * r + 8])
        g.replay()
        for s in range(8):
            eager.act(acts[8 * r + s])
        re_, oe, fe_first = eager.observe()
        rg, og, fg_first = graph.observe()
        assert torch.equal(oe["rgb"], og["rgb"]) and torch.equal(re_, rg) and torch.equal(fe_first, fg_first), f"replay {r}"
        assert torch.equal(fe["level_end"], fg["level_end"]), f"replay {r}: level_end"
        assert torch.equal(fe["rgb"], fg["rgb"]), f"replay {r}: final frames"
        ends += int((fe["level_end"] != 0).sum())
    assert ends > 0
    assert eager.errors() == 0 and graph.errors() == 0
    eager.close()
    graph.close()


def test_python_accessor_rules(product_lib):
    """The tensors alias the library's arrays (the same ones on every call); the first call is refused inside a
    capture; kernel timing is refused on a handle with final outputs."""
    import torch

    from procgen_b200 import ProcgenGym3Env

    kw = dict(distribution_mode="easy", num_levels=0, start_level=0, rand_seed=0, resource_root=STANDIN_PACK)
    env = ProcgenGym3Env(64, "coinrun", **kw)
    other = ProcgenGym3Env(64, "coinrun", **kw)
    a = torch.zeros(64, dtype=torch.int32, device="cuda")
    g = torch.cuda.CUDAGraph()
    with pytest.raises(RuntimeError, match="final_outputs"):
        with torch.cuda.graph(g):
            other.final_outputs()
    out = env.final_outputs()
    assert out["rgb"].shape == (64, 64, 64, 3) and out["rgb"].dtype == torch.uint8 and out["level_end"].shape == (64,)
    again = env.final_outputs()
    assert again["rgb"].data_ptr() == out["rgb"].data_ptr() and again["level_end"].data_ptr() == out["level_end"].data_ptr()
    with pytest.raises(RuntimeError):
        env.kernel_timing_begin(16)
    a[:8] = -1
    env.act(a)
    _, ob, first = env.observe()
    assert out["level_end"][:8].tolist() == [3] * 8 and bool(first[:8].all())
    assert env.errors() == 0
    env.close()
    other.close()
