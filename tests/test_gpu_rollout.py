"""The rollout (pgb200_get_rollout, env.rollout()) on the GPU, through the device-resident Python API.

At benchmark size, with final outputs, the pause mask and the consumer output on as well: a handle with the rollout and
an untouched control step together, and after every step their outputs are equal and every slot of the ring holds the
outputs of the step that wrote it, which the test keeps as a learner would (a copy of each step's outputs). Then a CUDA
graph of 8 steps replayed across wraps of the ring, host-buffer handles, and the device memory given back at close."""
import numpy as np
import pytest

from oracle.record import STANDIN_PACK

pytestmark = pytest.mark.gpu

ALL16 = "bigfish,bossfight,caveflyer,chaser,climber,coinrun,dodgeball,fruitbot,heist,jumper,leaper,maze,miner,ninja,plunder,starpilot"


class Expected:
    """What each slot of a rollout must hold: a copy of the outputs of the step that wrote it"""

    def __init__(self, roll, rew, rgb, first):
        self.slots = roll["rgb"].shape[0]
        self.rgb = roll["rgb"].clone()
        self.rew = roll["rew"].clone()
        self.first = roll["first"].clone()
        self.c = 0
        self.store(rew, rgb, first)

    def store(self, rew, rgb, first):
        self.rgb[self.c].copy_(rgb)
        self.rew[self.c].copy_(rew)
        self.first[self.c].copy_(first.to(self.first.dtype))

    def step(self, rew, rgb, first):
        self.c = (self.c + 1) % self.slots
        self.store(rew, rgb, first)

    def check(self, roll, what):
        import torch

        assert int(roll["cursor"].item()) == self.c, f"{what}: cursor {int(roll['cursor'].item())}, expected {self.c}"
        for s in range(self.slots):
            assert torch.equal(roll["rgb"][s], self.rgb[s]), f"{what}: slot {s} rgb (cursor {self.c})"
            assert torch.equal(roll["rew"][s], self.rew[s]), f"{what}: slot {s} rew"
            assert torch.equal(roll["first"][s], self.first[s]), f"{what}: slot {s} first"


def _with_everything(n, name, seed):
    import torch

    from procgen_b200 import ProcgenGym3Env

    kw = dict(distribution_mode="easy" if name == "coinrun" else "hard", num_levels=0, start_level=0, rand_seed=seed,
              resource_root=STANDIN_PACK)
    env = ProcgenGym3Env(n, name, **kw)
    env.final_outputs()
    env.pause_mask()
    env.enable_consumer_output(torch.float16, 2)
    return env


@pytest.mark.parametrize("n,name", [(65536, "coinrun"), (32768, ALL16)])
def test_full_size_against_a_control(product_lib, n, name):
    import torch

    slots = 4
    ctl, dut = _with_everything(n, name, 3), _with_everything(n, name, 3)
    gen = torch.Generator(device="cuda").manual_seed(1)
    warm = torch.randint(0, 15, (n,), device="cuda", dtype=torch.int32, generator=gen)
    for env in (ctl, dut):
        env.act(warm)
    roll = dut.rollout(slots)
    assert roll["rgb"].shape == (slots, n, 64, 64, 3) and roll["rew"].shape == (slots, n) and roll["cursor"].shape == (1,)
    rew, ob, first = dut.observe()
    exp = Expected(roll, rew, ob["rgb"], first)
    exp.check(roll, "the first call")
    paused = ended = 0
    for t in range(slots + 3):
        a = torch.randint(0, 15, (n,), device="cuda", dtype=torch.int32, generator=gen)
        a[torch.rand(n, device="cuda", generator=gen) < 0.05] = -1  # resets by the caller, beside the games' own
        m =(torch.rand(n, device="cuda", generator=gen) < 0.3).to(torch.uint8)
        for env in (ctl, dut):
            env.pause_mask().copy_(m)
            env.act(a)
        r1, o1, f1 = ctl.observe()
        r2, o2, f2 = dut.observe()
        assert torch.equal(o1["rgb"], o2["rgb"]) and torch.equal(r1, r2) and torch.equal(f1, f2), f"step {t}"
        for key, v in ctl.get_info_tensors().items():
            assert torch.equal(v, dut.get_info_tensors()[key]), f"step {t}: info {key}"
        fc, fd = ctl.final_outputs(), dut.final_outputs()
        assert torch.equal(fc["level_end"], fd["level_end"]) and torch.equal(fc["rgb"], fd["rgb"]), f"step {t}: final outputs"
        assert torch.equal(ctl.consumer_observation(), dut.consumer_observation()), f"step {t}: consumer output"
        exp.step(r2, o2["rgb"], f2)
        exp.check(roll, f"step {t}")
        paused += int(m.sum())
        ended += int((fd["level_end"] != 0).sum())
    assert paused > 0 and ended > 0
    assert ctl.errors() == 0 and dut.errors() == 0
    ctl.close()
    dut.close()


def test_graph_replayed_across_wraps(product_lib):
    """A graph of 8 act() calls replayed: the rollout holds the outputs of the last `slots` eager steps of a control.
    The first rollout() call is refused inside a capture; a second one is not."""
    import torch

    from procgen_b200 import ProcgenGym3Env

    n, reps, slots = 4096, 4, 5
    kw = dict(distribution_mode="hard", num_levels=0, start_level=0, rand_seed=5, resource_root=STANDIN_PACK)
    other = ProcgenGym3Env(64, "coinrun", **kw)
    with pytest.raises(RuntimeError, match="rollout"):
        with torch.cuda.graph(torch.cuda.CUDAGraph()):
            other.rollout(slots)
    other.close()
    eager = ProcgenGym3Env(n, "bigfish,coinrun", **kw)
    graph = ProcgenGym3Env(n, "bigfish,coinrun", **kw)
    roll = graph.rollout(slots)
    rew, ob, first = eager.observe()
    exp = Expected(roll, rew, ob["rgb"], first)
    gen = torch.Generator(device="cuda").manual_seed(4)
    acts = torch.randint(-1, 15, (reps * 8, n), device="cuda", dtype=torch.int32, generator=gen)
    abuf = torch.zeros((8, n), device="cuda", dtype=torch.int32)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for s in range(8):
            graph.act(abuf[s])
        again = graph.rollout(slots)
    assert again["rgb"].data_ptr() == roll["rgb"].data_ptr()
    torch.cuda.synchronize()
    exp.check(roll, "after the capture")
    for r in range(reps):
        abuf.copy_(acts[8 * r:8 * r + 8])
        g.replay()
        for s in range(8):
            eager.act(acts[8 * r + s])
            re_, oe, fe = eager.observe()
            exp.step(re_, oe["rgb"], fe)
        rg, og, fg = graph.observe()
        assert torch.equal(oe["rgb"], og["rgb"]) and torch.equal(re_, rg) and torch.equal(fe, fg), f"replay {r}"
        exp.check(roll, f"replay {r}")
    assert eager.errors() == 0 and graph.errors() == 0
    eager.close()
    graph.close()


def test_host_buffers(product_lib):
    """host_buffers=True: the rollout is complete once observe() returns, and holds what observe() returned."""
    import torch

    from procgen_b200 import ProcgenGym3Env

    n, slots = 512, 3
    kw = dict(distribution_mode="hard", num_levels=0, start_level=0, rand_seed=6, resource_root=STANDIN_PACK)
    host = ProcgenGym3Env(n, "bigfish,coinrun", host_buffers=True, **kw)
    dev = ProcgenGym3Env(n, "bigfish,coinrun", **kw)
    roll = host.rollout(slots)
    assert roll["rgb"].is_cuda and roll["rgb"].shape == (slots, n, 64, 64, 3)
    gen = torch.Generator(device="cuda").manual_seed(9)
    for t in range(3 * slots + 1):
        a = torch.randint(-1, 15, (n,), device="cuda", dtype=torch.int32, generator=gen)
        host.act(a.cpu().numpy())
        dev.act(a)
        r1, o1, f1 = host.observe()
        r2, o2, f2 = dev.observe()
        assert np.array_equal(r1, r2.cpu().numpy()) and np.array_equal(f1, f2.cpu().numpy()), f"step {t}"
        assert np.array_equal(o1["rgb"], o2["rgb"].cpu().numpy()), f"step {t}: rgb"
        c = int(roll["cursor"].item())
        assert c == (t + 1) % slots
        assert np.array_equal(roll["rgb"][c].cpu().numpy(), o1["rgb"]), f"step {t}: slot rgb"
        assert np.array_equal(roll["rew"][c].cpu().numpy(), r1) and np.array_equal(roll["first"][c].cpu().numpy(), f1.astype(np.uint8))
    host.close()
    dev.close()


def test_close_returns_device_memory(product_lib):
    """As tests/test_handle_lifetime.py, with the rollout on (48 KiB per env here)."""
    pynvml = pytest.importorskip("pynvml")
    import torch

    from oracle.ref_env import mt19937_actions
    from procgen_b200 import ProcgenGym3Env
    from test_handle_lifetime import NUM, _process_device_bytes

    def cycle():
        env = ProcgenGym3Env(NUM, "coinrun", distribution_mode="easy", num_levels=0, rand_seed=0, resource_root=STANDIN_PACK)
        env.rollout(4)
        for actions in mt19937_actions(0, NUM, 5):
            env.act(torch.as_tensor(actions, device="cuda"))
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
