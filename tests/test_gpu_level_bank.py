"""The level bank (pgb200_build_level_bank) on the GPU.

A bank changes nothing but speed, so existing records check it: banked handles replay the num_levels = 200 cases of
test_gpu_parity.py (every reset a bank hit, in host-buffer mode) and the 42 (game, mode) pairs of the level sweep
with the bank built over the sweep's own seeds (every swept level comes out of the bank), against the same records.
At benchmark size a banked handle runs in lockstep with an unbanked control through the device-resident Python API:
65 536 envs of the slow level generators, the 16-game list, final outputs, the pause mask, a CUDA graph with the bank
rebuilt in place between replays, and host-buffer mode."""
import ctypes as C

import numpy as np
import pytest

from helpers import make_checked_pair, run_lockstep
from level_bank import bank_info, build_bank
from level_sweep import LEVEL_SWEEP_RECORDS, PAIRS, run_level_sweep, sweep_seeds
from oracle.record import STANDIN_PACK, use_records
from oracle.ref_env import MAX_STATE_SIZE

pytestmark = pytest.mark.gpu

ALL16 = "bigfish,bossfight,caveflyer,chaser,climber,coinrun,dodgeball,fruitbot,heist,jumper,leaper,maze,miner,ninja,plunder,starpilot"
KW = dict(num_levels=200, start_level=0, rand_seed=0)

# test_gpu_parity.py::test_libenv_host_buffers_bit_exact, whose records these cases replay
HOST_BUFFER_CASES = [
    ("coinrun", "easy", 64, 1000), ("coinrun", "hard", 64, 1000), ("bigfish", "hard", 64, 1000), ("maze", "hard", 64, 800),
    ("heist", "hard", 64, 800), ("miner", "hard", 32, 600), ("leaper", "hard", 32, 600), ("plunder", "hard", 32, 800),
    ("chaser", "hard", 32, 600), ("climber", "hard", 32, 600), ("ninja", "hard", 32, 800), ("fruitbot", "hard", 32, 600),
    ("caveflyer", "hard", 32, 600), ("bossfight", "hard", 32, 800), ("dodgeball", "hard", 32, 600),
    ("starpilot", "hard", 32, 800), ("jumper", "hard", 32, 600), ("jumper", "easy", 32, 600),
]


@pytest.fixture(autouse=True, scope="module")
def _sweep_records():
    use_records(LEVEL_SWEEP_RECORDS)


@pytest.mark.parametrize("name,mode,n,steps", HOST_BUFFER_CASES)
def test_parity_records_with_a_bank(product_lib, name, mode, n, steps):
    key = f"test_gpu_parity.py::test_libenv_host_buffers_bit_exact[{name}-{mode}-{n}-{steps}]#0"
    ref, dut = make_checked_pair(product_lib, n, name, key=key, distribution_mode=mode, **KW)
    assert build_bank(dut, range(200)) == 0
    run_lockstep(ref, dut, steps)
    ref.close()
    dut.close()


def test_sixteen_game_list_records_with_a_bank(product_lib):
    key = "test_gpu_parity.py::test_sixteen_game_list_bit_exact#0"
    ref, dut = make_checked_pair(product_lib, 64, ALL16, key=key, distribution_mode="hard", **KW)
    assert build_bank(dut, range(200)) == 0
    run_lockstep(ref, dut, 500)
    ref.close()
    dut.close()


@pytest.mark.parametrize("name,mode", PAIRS)
def test_level_sweep_out_of_the_bank(product_lib, name, mode):
    seeds = sweep_seeds(name, mode, 1024)
    key = f"test_gpu_level_sweep.py::test_level_sweep[{name}-{mode}]#0"
    ref, dut = make_checked_pair(product_lib, 256, name, key=key, distribution_mode=mode, num_levels=0, start_level=0, rand_seed=0)
    assert build_bank(dut, seeds) == 0
    assert bank_info(dut)[0] == len(set(seeds))
    assert run_level_sweep(ref, dut, seeds, 24) == 4
    ref.close()
    dut.close()


# ------------------------------------------------------------------ banked against an unbanked control
def _blob(env, e, buf=C.create_string_buffer(MAX_STATE_SIZE)):
    k = int(env._lib.get_state(env._h, int(e), buf, MAX_STATE_SIZE))
    return bytes(buf.raw[:k])


def _pair(name, n, mode="hard", **extra):
    from procgen_b200 import ProcgenGym3Env

    kw = dict(KW, distribution_mode=mode, resource_root=STANDIN_PACK, **extra)
    ctl, banked = ProcgenGym3Env(n, name, **kw), ProcgenGym3Env(n, name, **kw)
    banked.build_level_bank()
    assert banked.level_bank_info()["levels"] == 200
    return ctl, banked


def _same_outputs(ctl, banked, t):
    import torch

    r1, o1, f1 = ctl.observe()
    r2, o2, f2 = banked.observe()
    assert torch.equal(r1, r2) and torch.equal(f1, f2), f"step {t}: rew / first differ"
    assert torch.equal(o1["rgb"], o2["rgb"]), f"step {t}: rgb differs at envs {(o1['rgb'] != o2['rgb']).flatten(1).any(1).nonzero()[:8].tolist()}"
    for k, v in ctl.get_info_tensors().items():
        assert torch.equal(v, banked.get_info_tensors()[k]), f"step {t}: info {k}"


def _picks(n):
    """256 envs spread over all 8 launch chunks of every game"""
    return [int(c * (n // 8) + j * (n // 8 // 32) + (c * 7 + j) % 16) for c in range(8) for j in range(32)]


@pytest.mark.parametrize("name,mode", [("coinrun", "easy"), ("caveflyer", "hard"), ("jumper", "hard"), ("leaper", "hard"), (ALL16, "hard")])
def test_full_size_lockstep_with_a_control(product_lib, name, mode):
    import torch

    n, steps = 65536, 150
    ctl, banked = _pair(name, n, mode)
    gen = torch.Generator(device="cuda").manual_seed(1)
    starts = 0
    for t in range(steps):
        a = torch.randint(0, 15, (n,), device="cuda", dtype=torch.int32, generator=gen)
        a[torch.rand(n, device="cuda", generator=gen) < 0.03] = -1
        ctl.act(a)
        banked.act(a)
        _same_outputs(ctl, banked, t)
        starts += int(ctl.observe()[2].sum())
        if t % 50 == 49:
            for e in _picks(n):
                assert _blob(ctl, e) == _blob(banked, e), f"step {t} env {e}: state blobs differ"
    assert starts > n, starts
    assert ctl.errors() == 0 and banked.errors() == 0
    ctl.close()
    banked.close()


def test_final_outputs_and_pause_mask_with_a_control(product_lib):
    import torch

    n = 8192
    ctl, banked = _pair(ALL16, n)
    fc, fb = ctl.final_outputs(), banked.final_outputs()
    mc, mb = ctl.pause_mask(), banked.pause_mask()
    gen = torch.Generator(device="cuda").manual_seed(2)
    for t in range(120):
        m = (torch.rand(n, device="cuda", generator=gen) < 0.3).to(torch.uint8)
        mc.copy_(m)
        mb.copy_(m)
        a = torch.randint(-1, 15, (n,), device="cuda", dtype=torch.int32, generator=gen)
        ctl.act(a)
        banked.act(a)
        _same_outputs(ctl, banked, t)
        assert torch.equal(fc["level_end"], fb["level_end"]), f"step {t}: level_end"
        ended = fc["level_end"] != 0
        assert torch.equal(fc["rgb"][ended], fb["rgb"][ended]), f"step {t}: final frames"
    for e in _picks(n):
        assert _blob(ctl, e) == _blob(banked, e), f"env {e}: state blobs differ"
    assert ctl.errors() == 0 and banked.errors() == 0
    ctl.close()
    banked.close()


def test_graph_sees_an_in_place_rebuild(product_lib):
    """A graph of 8 steps captured on a banked handle, replayed with the bank rebuilt in place between replays
    (other seeds, then empty, then the full range again): equal to eager steps of an unbanked control. Nothing in
    the loop waits for the device: each replay's outputs are cloned on the stream, and all are compared at the end,
    so a rebuild that were not ordered behind the replay before it would race with it. Both calls are refused
    inside a capture."""
    import torch

    n, reps = 4096, 6
    ctl, banked = _pair("caveflyer,jumper", n)
    with pytest.raises(RuntimeError, match="build_level_bank"):
        with torch.cuda.graph(torch.cuda.CUDAGraph()):
            banked.build_level_bank()
    with pytest.raises(RuntimeError, match="level_bank_info"):
        with torch.cuda.graph(torch.cuda.CUDAGraph()):
            banked.level_bank_info()
    gen = torch.Generator(device="cuda").manual_seed(4)
    acts = torch.randint(-1, 15, (reps * 8, n), device="cuda", dtype=torch.int32, generator=gen)
    abuf = torch.zeros((8, n), device="cuda", dtype=torch.int32)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for s in range(8):
            banked.act(abuf[s])
    torch.cuda.synchronize()
    banks = [range(200), range(0, 200, 2), [], range(100, 300), range(200), range(200)]

    def snapshot(env):
        rew, ob, first = env.observe()
        return [rew.clone(), ob["rgb"].clone(), first.clone()] + [v.clone() for v in env.get_info_tensors().values()]

    got, want = [], []
    for r in range(reps):
        banked.build_level_bank(banks[r], capacity=0)
        abuf.copy_(acts[8 * r:8 * r + 8])
        g.replay()
        got.append(snapshot(banked))
        for s in range(8):
            ctl.act(acts[8 * r + s])
        want.append(snapshot(ctl))
    torch.cuda.synchronize()
    for r in range(reps):
        for k, (a, b) in enumerate(zip(want[r], got[r])):
            assert torch.equal(a, b), f"replay {r}: output {k} differs"
    for e in range(0, n, 97):
        assert _blob(ctl, e) == _blob(banked, e), f"env {e}: state blobs differ"
    assert ctl.errors() == 0 and banked.errors() == 0
    ctl.close()
    banked.close()


def test_host_buffer_mode(product_lib):
    from procgen_b200 import ProcgenGym3Env

    n = 512
    kw = dict(KW, distribution_mode="hard", resource_root=STANDIN_PACK, host_buffers=True)
    ctl, banked = ProcgenGym3Env(n, ALL16, **kw), ProcgenGym3Env(n, ALL16, **kw)
    banked.build_level_bank()
    with pytest.raises(ValueError):
        banked.build_level_bank(range(201))
    rs = np.random.RandomState(5)
    for t in range(100):
        a = rs.randint(-1, 15, size=n).astype(np.int32)
        ctl.act(a)
        banked.act(a)
        r1, o1, f1 = ctl.observe()
        r2, o2, f2 = banked.observe()
        assert np.array_equal(r1, r2) and np.array_equal(f1, f2) and np.array_equal(o1["rgb"], o2["rgb"]), f"step {t}"
    info = banked.level_bank_info()
    assert info["levels"] == 200 and info["bytes"] > 0
    ctl.close()
    banked.close()
