"""Level lookahead (pgb200_enable_level_lookahead) on the GPU.

Lookahead changes nothing but speed, so existing records check it: lookahead handles replay the host-buffer cases of
test_gpu_parity.py and its 16-game list against the same records, and their counters must show resets served from
the slots. At benchmark size a lookahead handle runs in lockstep with a control without it through the
device-resident Python API at num_levels = 0: 65 536 envs of the slow level generators, coinrun and the 16-game list;
final outputs, the pause mask and the consumer ring; an 8-step CUDA graph captured after enable; host-buffer mode.
Where nothing can make a prediction miss, no reset may generate. A closed handle gives its device memory back."""
import ctypes as C

import numpy as np
import pytest

from helpers import make_checked_pair, run_lockstep
from level_lookahead import enable_lookahead, lookahead_info
from oracle.record import STANDIN_PACK
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


@pytest.mark.parametrize("name,mode,n,steps", HOST_BUFFER_CASES)
def test_parity_records_with_lookahead(product_lib, name, mode, n, steps):
    key = f"test_gpu_parity.py::test_libenv_host_buffers_bit_exact[{name}-{mode}-{n}-{steps}]#0"
    ref, dut = make_checked_pair(product_lib, n, name, key=key, distribution_mode=mode, **KW)
    assert enable_lookahead(dut) == 0
    run_lockstep(ref, dut, steps)
    info = lookahead_info(dut)
    assert info["served"] > 0 and info["generated"] == 0, info
    ref.close()
    dut.close()


def test_sixteen_game_list_records_with_lookahead(product_lib):
    key = "test_gpu_parity.py::test_sixteen_game_list_bit_exact#0"
    ref, dut = make_checked_pair(product_lib, 64, ALL16, key=key, distribution_mode="hard", **KW)
    assert enable_lookahead(dut) == 0
    run_lockstep(ref, dut, 500)
    info = lookahead_info(dut)
    assert info["served"] > 64 and info["generated"] == 0, info
    ref.close()
    dut.close()


# ------------------------------------------------------------------ against a control without lookahead
def _blob(env, e, buf=C.create_string_buffer(MAX_STATE_SIZE)):
    k = int(env._lib.get_state(env._h, int(e), buf, MAX_STATE_SIZE))
    return bytes(buf.raw[:k])


def _pair(name, n, mode="hard", **extra):
    from procgen_b200 import ProcgenGym3Env

    kw = dict(distribution_mode=mode, num_levels=0, start_level=0, rand_seed=0, resource_root=STANDIN_PACK, **extra)
    ctl, look = ProcgenGym3Env(n, name, **kw), ProcgenGym3Env(n, name, **kw)
    look.enable_level_lookahead()
    look.enable_level_lookahead()  # a second call does nothing
    assert look.level_lookahead_info()["bytes"] > 0
    return ctl, look


def _same_outputs(ctl, look, t):
    import torch

    r1, o1, f1 = ctl.observe()
    r2, o2, f2 = look.observe()
    assert torch.equal(r1, r2) and torch.equal(f1, f2), f"step {t}: rew / first differ"
    assert torch.equal(o1["rgb"], o2["rgb"]), f"step {t}: rgb differs at envs {(o1['rgb'] != o2['rgb']).flatten(1).any(1).nonzero()[:8].tolist()}"
    for k, v in ctl.get_info_tensors().items():
        assert torch.equal(v, look.get_info_tensors()[k]), f"step {t}: info {k}"


def _picks(n):
    """256 envs spread over all 8 launch chunks of every game"""
    return [int(c * (n // 8) + j * (n // 8 // 32) + (c * 7 + j) % 16) for c in range(8) for j in range(32)]


@pytest.mark.parametrize("name,mode", [("caveflyer", "hard"), ("jumper", "hard"), ("leaper", "hard"), ("coinrun", "easy"), (ALL16, "hard")])
def test_full_size_lockstep_with_a_control(product_lib, name, mode):
    import torch

    n, steps = 65536, 100
    ctl, look = _pair(name, n, mode)
    gen = torch.Generator(device="cuda").manual_seed(1)
    resets = 0
    for t in range(steps):
        a = torch.randint(0, 15, (n,), device="cuda", dtype=torch.int32, generator=gen)
        a[torch.rand(n, device="cuda", generator=gen) < 0.03] = -1
        ctl.act(a)
        look.act(a)
        _same_outputs(ctl, look, t)
        resets += int(ctl.observe()[2].sum())
        if t % 25 == 24:
            for e in _picks(n):
                assert _blob(ctl, e) == _blob(look, e), f"step {t} env {e}: state blobs differ"
    info = look.level_lookahead_info()
    assert resets > n and info["served"] == resets and info["generated"] == 0 and info["bank"] == 0, (resets, info)
    assert ctl.errors() == 0 and look.errors() == 0
    ctl.close()
    look.close()


def test_final_outputs_pause_mask_and_consumer_ring_with_a_control(product_lib):
    import torch

    n = 8192
    ctl, look = _pair(ALL16, n)
    fc, fl = ctl.final_outputs(), look.final_outputs()
    mc, ml = ctl.pause_mask(), look.pause_mask()
    for env in (ctl, look):
        env.enable_consumer_output(torch.float16, 4)
    gen = torch.Generator(device="cuda").manual_seed(2)
    ends = 0
    for t in range(120):
        m = (torch.rand(n, device="cuda", generator=gen) < 0.3).to(torch.uint8)
        mc.copy_(m)
        ml.copy_(m)
        a = torch.randint(-1, 15, (n,), device="cuda", dtype=torch.int32, generator=gen)
        ctl.act(a)
        look.act(a)
        _same_outputs(ctl, look, t)
        assert torch.equal(fc["level_end"], fl["level_end"]), f"step {t}: level_end"
        ended = fc["level_end"] != 0
        ends += int(ended.sum())
        assert torch.equal(fc["rgb"][ended], fl["rgb"][ended]), f"step {t}: final frames"
        assert torch.equal(ctl.consumer_observation(), look.consumer_observation()), f"step {t}: consumer stacks"
    for e in _picks(n):
        assert _blob(ctl, e) == _blob(look, e), f"env {e}: state blobs differ"
    info = look.level_lookahead_info()
    assert ends > n and info["served"] == ends and info["generated"] == 0, (ends, info)
    assert ctl.errors() == 0 and look.errors() == 0
    ctl.close()
    look.close()


def test_graph_captured_after_enable(product_lib):
    """8 steps captured after enable_level_lookahead and replayed: equal to eager steps of a control, with every
    reset of the replays served from the slots. Both methods are refused inside a capture."""
    import torch

    n, reps = 8192, 6
    ctl, look = _pair("caveflyer,jumper,leaper,coinrun", n)
    for method in ("enable_level_lookahead", "level_lookahead_info"):
        with pytest.raises(RuntimeError, match=method):
            with torch.cuda.graph(torch.cuda.CUDAGraph()):
                getattr(look, method)()
    gen = torch.Generator(device="cuda").manual_seed(4)
    acts = torch.randint(-1, 15, (reps * 8, n), device="cuda", dtype=torch.int32, generator=gen)
    abuf = torch.zeros((8, n), device="cuda", dtype=torch.int32)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for s in range(8):
            look.act(abuf[s])
    torch.cuda.synchronize()
    before = look.level_lookahead_info()

    def snapshot(env):
        rew, ob, first = env.observe()
        return [rew.clone(), ob["rgb"].clone(), first.clone()] + [v.clone() for v in env.get_info_tensors().values()]

    got, want, resets = [], [], 0
    for r in range(reps):
        abuf.copy_(acts[8 * r:8 * r + 8])
        g.replay()
        got.append(snapshot(look))
        for s in range(8):
            ctl.act(acts[8 * r + s])
            resets += int(ctl.observe()[2].sum())
        want.append(snapshot(ctl))
    torch.cuda.synchronize()
    for r in range(reps):
        for k, (a, b) in enumerate(zip(want[r], got[r])):
            assert torch.equal(a, b), f"replay {r}: output {k} differs"
    for e in range(0, n, 97):
        assert _blob(ctl, e) == _blob(look, e), f"env {e}: state blobs differ"
    after = look.level_lookahead_info()
    assert after["served"] - before["served"] == resets > 0 and after["generated"] == 0, (resets, before, after)
    assert ctl.errors() == 0 and look.errors() == 0
    ctl.close()
    look.close()


def test_host_buffer_mode(product_lib):
    from procgen_b200 import ProcgenGym3Env

    n = 512
    kw = dict(distribution_mode="hard", num_levels=0, rand_seed=0, resource_root=STANDIN_PACK, host_buffers=True)
    ctl, look = ProcgenGym3Env(n, ALL16, **kw), ProcgenGym3Env(n, ALL16, **kw)
    look.enable_level_lookahead()
    rs = np.random.RandomState(5)
    resets = 0
    for t in range(100):
        a = rs.randint(-1, 15, size=n).astype(np.int32)
        ctl.act(a)
        look.act(a)
        r1, o1, f1 = ctl.observe()
        r2, o2, f2 = look.observe()
        assert np.array_equal(r1, r2) and np.array_equal(f1, f2) and np.array_equal(o1["rgb"], o2["rgb"]), f"step {t}"
        resets += int(f1.sum())
    info = look.level_lookahead_info()
    assert info["served"] == resets and info["generated"] == 0, (resets, info)
    ctl.close()
    look.close()


def test_close_returns_device_memory(product_lib):
    """As tests/test_handle_lifetime.py, with lookahead on (its slots are the largest arrays of such a handle): the
    process's device memory does not grow across two cycles by a 2 MiB page, the unit NVML counts in."""
    pynvml = pytest.importorskip("pynvml")
    import torch

    from oracle.ref_env import mt19937_actions
    from procgen_b200 import ProcgenGym3Env
    from test_handle_lifetime import _process_device_bytes

    num = 4096

    def cycle():
        env = ProcgenGym3Env(num, "coinrun", distribution_mode="easy", num_levels=0, rand_seed=0, resource_root=STANDIN_PACK)
        env.build_level_bank([1, 2, 3])
        env.enable_level_lookahead()
        for actions in mt19937_actions(0, num, 3):
            actions[::7] = -1
            env.act(torch.as_tensor(actions, device="cuda"))
            env.observe()
        env.close()
        del env
        torch.cuda.synchronize()
        torch.cuda.empty_cache()

    pynvml.nvmlInit()
    try:
        cycle()
        before = _process_device_bytes(pynvml)
        if before is None:
            pytest.skip("NVML does not list this process (PID namespace)")
        cycle()
        cycle()
        after = _process_device_bytes(pynvml)
    finally:
        pynvml.nvmlShutdown()
    assert after - before < 2 << 20, f"two handles left {after - before} bytes of device memory behind"
