"""Action repeat (pgb200_get_action_repeat) on the GPU, through the device-resident Python API.

A step with repeat counts equals single steps of a control handle without them: the control steps up to max(r) times
with the same actions, and pauses each env (its pause mask) once its level has ended or it has used its count. The
control's rewards are summed with torch in float32; its first, infos and frames are those of each env's last game
step. Frames, outputs, final outputs, the rollout, the consumer output and state blobs are compared."""
import numpy as np
import pytest

from oracle.record import STANDIN_PACK

pytestmark = pytest.mark.gpu

ALL16 = "bigfish,bossfight,caveflyer,chaser,climber,coinrun,dodgeball,fruitbot,heist,jumper,leaper,maze,miner,ninja,plunder,starpilot"


def _env(n, name, **kw):
    from procgen_b200 import ProcgenGym3Env

    return ProcgenGym3Env(n, name, **dict(dict(distribution_mode="hard", num_levels=0, start_level=0, rand_seed=0,
                                                resource_root=STANDIN_PACK), **kw))


class Control:
    """A handle without action repeat that plays another handle's repeated steps one game step at a time"""

    def __init__(self, env, final=False):
        import torch

        self.env = env
        self.mask = env.pause_mask()
        n = env.num
        self.rew = torch.zeros(n, dtype=torch.float32, device="cuda")
        self.first = torch.zeros(n, dtype=torch.bool, device="cuda")
        self.level_end = torch.zeros(n, dtype=torch.uint8, device="cuda") if final else None

    def step(self, actions, reps, paused=None):
        """The control's version of one act(actions) with counts `reps` and pause mask `paused` (bool, or None).
        Returns the game steps each env played."""
        import torch

        n = self.env.num
        count = reps.clamp(min=1)
        live = torch.ones(n, dtype=torch.bool, device="cuda") if paused is None else ~paused
        played = torch.zeros(n, dtype=torch.int32, device="cuda")
        self.rew.zero_()
        self.first.zero_()
        if self.level_end is not None:
            self.level_end.zero_()
        while bool(live.any()):
            self.mask.copy_((~live).to(torch.uint8))
            self.env.act(actions)
            rew, _, first = self.env.observe()
            self.rew = torch.where(live, self.rew + rew, self.rew)
            self.first = torch.where(live, first, self.first)
            if self.level_end is not None:
                self.level_end = torch.where(live, self.env.final_outputs()["level_end"], self.level_end)
            ended = first | (self.env.get_info_tensors()["prev_level_complete"] != 0)
            played += live.to(torch.int32)
            live &= ~ended & (played < count)
        return played


def _assert_same(dut, ctl, t, final=False):
    import torch

    rew, ob, first = dut.observe()
    _, cob, _ = ctl.env.observe()
    bad = (ob["rgb"] != cob["rgb"]).flatten(1).any(1)
    assert not bool(bad.any()), f"step {t}: rgb differs at envs {bad.nonzero()[:8].flatten().tolist()}"
    assert torch.equal(rew, ctl.rew), f"step {t}: rew differs at envs {(rew != ctl.rew).nonzero()[:8].flatten().tolist()}"
    assert torch.equal(first, ctl.first), f"step {t}: first differs"
    for k, v in dut.get_info_tensors().items():
        assert torch.equal(v, ctl.env.get_info_tensors()[k]), f"step {t}: info {k}"
    if final:
        fd, fc = dut.final_outputs(), ctl.env.final_outputs()
        assert torch.equal(fd["level_end"], ctl.level_end), f"step {t}: level_end"
        assert torch.equal(fd["rgb"], fc["rgb"]), f"step {t}: final frames"


def _assert_same_blobs(dut, ctl, envs):
    for e, a, b in zip(envs, dut.get_state(envs), ctl.env.get_state(envs)):
        assert a == b, f"env {e}: state blobs differ"


def _run(n, name, steps, choices, seed, blob_envs=256, **kw):
    import torch

    dut, ctl = _env(n, name, **kw), Control(_env(n, name, **kw))
    rep = dut.action_repeat()
    assert rep.dtype == torch.int32 and bool((rep == 1).all())
    gen = torch.Generator(device="cuda").manual_seed(seed)
    choices = torch.as_tensor(choices, dtype=torch.int32, device="cuda")
    picks = np.random.RandomState(seed).choice(n, size=min(n, blob_envs), replace=False).tolist()
    most = 0
    for t in range(steps):
        r = choices[torch.randint(len(choices), (n,), device="cuda", generator=gen)]
        a = torch.randint(0, 15, (n,), device="cuda", dtype=torch.int32, generator=gen)
        a[torch.rand(n, device="cuda", generator=gen) < 0.03] = -1
        rep.copy_(r)
        dut.act(a)
        most = max(most, int(ctl.step(a, r).max()))
        _assert_same(dut, ctl, t)
        if t % 10 == 9:
            _assert_same_blobs(dut, ctl, picks)
    assert most > 1
    assert dut.errors() == 0 and ctl.env.errors() == 0
    dut.close()
    ctl.env.close()


def test_coinrun_easy_65536(product_lib):
    _run(65536, "coinrun", 30, [-1, 0, 1, 2, 4, 8], 1, distribution_mode="easy")


def test_sixteen_game_list_32768(product_lib):
    _run(32768, ALL16, 30, [1, 2, 3, 4, 6], 2)


@pytest.mark.parametrize("name", ["coinrun", "jumper"])
def test_whole_world_view(product_lib, name):
    _run(4096, name, 30, [0, 1, 2, 5], 3, center_agent=False)


def test_every_opt_in(product_lib):
    """Level choice, final outputs, the pause mask, the level bank, lookahead, a 3-slot rollout and a 4-frame consumer
    output on the 16-game list. The rollout's slot of each step holds the step's summed rew, last frame and first; the
    consumer stack is the control's last frames, stacked by the usual rule."""
    import torch

    n, slots, k = 4096, 3, 4
    kw = dict(num_levels=64)
    dut, ctl_env = _env(n, ALL16, **kw), _env(n, ALL16, **kw)
    ctl = Control(ctl_env, final=True)
    for env in (dut, ctl_env):
        env.next_level_seeds()
        env.final_outputs()
        env.build_level_bank(list(range(32)))
    dut.enable_level_lookahead()
    roll = dut.rollout(slots)
    dut.enable_consumer_output(torch.float16, frames=k)
    rep, mask = dut.action_repeat(), dut.pause_mask()
    gen = torch.Generator(device="cuda").manual_seed(4)
    dt = torch.float16

    def frame(env):
        return (env.observe()[1]["rgb"].permute(0, 3, 1, 2).float() / 255.0).to(dt)

    stack = torch.zeros((n, k, 3, 64, 64), dtype=dt, device="cuda")
    stack[:, -1] = frame(dut)
    picks = np.random.RandomState(4).choice(n, size=256, replace=False).tolist()
    for t in range(40):
        r = torch.randint(-1, 7, (n,), device="cuda", dtype=torch.int32, generator=gen)
        a = torch.randint(0, 15, (n,), device="cuda", dtype=torch.int32, generator=gen)
        a[torch.rand(n, device="cuda", generator=gen) < 0.05] = -1
        paused = torch.rand(n, device="cuda", generator=gen) < 0.2
        seeds = torch.where(torch.rand(n, device="cuda", generator=gen) < 0.3,
                            torch.randint(0, 64, (n,), device="cuda", dtype=torch.int32, generator=gen), -1)
        for env in (dut, ctl_env):
            env.next_level_seeds().copy_(seeds)
        rep.copy_(r)
        mask.copy_(paused.to(torch.uint8))
        cursor = int(roll["cursor"][0])
        dut.act(a)
        ctl.step(a, r, paused)
        _assert_same(dut, ctl, t, final=True)
        assert torch.equal(dut.next_level_seeds(), ctl_env.next_level_seeds()), f"step {t}: override array"
        rew, ob, first = dut.observe()
        c = int(roll["cursor"][0])
        assert c == (cursor + 1) % slots, f"step {t}: the rollout moved on {c - cursor} slots"
        assert torch.equal(roll["rgb"][c], ob["rgb"]) and torch.equal(roll["rew"][c], rew), f"step {t}: rollout slot"
        assert torch.equal(roll["first"][c], first.to(torch.uint8)), f"step {t}: rollout first"
        stack = torch.cat([stack[:, 1:], frame(ctl_env)[:, None]], 1)
        stack[ctl.first, :-1] = 0
        got = dut.consumer_observation().reshape(n, k, 3, 64, 64)
        assert torch.equal(got, stack), f"step {t}: consumer stacks differ"
        if t % 10 == 9:
            _assert_same_blobs(dut, ctl, picks)
    assert bool((rep >= -1).all()) and int(mask.sum()) > 0
    assert dut.errors() == 0 and ctl_env.errors() == 0
    dut.close()
    ctl_env.close()


def test_graph_with_the_counts_refilled_inside(product_lib):
    """A graph of 8 act() calls, each behind a copy into the counts, replayed: equal to eager steps with the same counts.
    The first action_repeat() call is refused inside a capture."""
    import torch

    n, reps = 4096, 6
    other = _env(64, "coinrun", rand_seed=5)
    with pytest.raises(RuntimeError, match="action_repeat"):
        with torch.cuda.graph(torch.cuda.CUDAGraph()):
            other.action_repeat()
    other.close()
    eager, graph = _env(n, "bigfish,coinrun", rand_seed=5), _env(n, "bigfish,coinrun", rand_seed=5)
    re_, rg = eager.action_repeat(), graph.action_repeat()
    gen = torch.Generator(device="cuda").manual_seed(4)
    acts = torch.randint(-1, 15, (reps * 8, n), device="cuda", dtype=torch.int32, generator=gen)
    counts = torch.randint(-1, 9, (reps * 8, n), device="cuda", dtype=torch.int32, generator=gen)
    abuf = torch.zeros((8, n), device="cuda", dtype=torch.int32)
    rbuf = torch.zeros((8, n), device="cuda", dtype=torch.int32)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for s in range(8):
            rg.copy_(rbuf[s])
            graph.act(abuf[s])
    torch.cuda.synchronize()
    for i in range(reps):
        abuf.copy_(acts[8 * i:8 * i + 8])
        rbuf.copy_(counts[8 * i:8 * i + 8])
        g.replay()
        for s in range(8):
            re_.copy_(counts[8 * i + s])
            eager.act(acts[8 * i + s])
        r1, o1, f1 = eager.observe()
        r2, o2, f2 = graph.observe()
        assert torch.equal(o1["rgb"], o2["rgb"]) and torch.equal(r1, r2) and torch.equal(f1, f2), f"replay {i}"
        for key, v in eager.get_info_tensors().items():
            assert torch.equal(v, graph.get_info_tensors()[key]), f"replay {i}: info {key}"
    picks = list(range(0, n, 61))
    assert eager.get_state(picks) == graph.get_state(picks)
    assert eager.errors() == 0 and graph.errors() == 0
    eager.close()
    graph.close()


def test_host_buffers(product_lib):
    """host_buffers=True: action_repeat() written with torch, act() waits for the writes; equal to the control"""
    import torch

    n = 256
    host = _env(n, "bigfish,coinrun", rand_seed=6, host_buffers=True)
    ctl = Control(_env(n, "bigfish,coinrun", rand_seed=6))
    rep = host.action_repeat()
    assert rep.is_cuda and rep.dtype == torch.int32 and rep.shape == (n,)
    gen = torch.Generator(device="cuda").manual_seed(9)
    for t in range(60):
        r = torch.randint(-1, 6, (n,), device="cuda", dtype=torch.int32, generator=gen)
        a = torch.randint(-1, 15, (n,), device="cuda", dtype=torch.int32, generator=gen)
        rep.copy_(r)
        host.act(a.cpu().numpy())
        ctl.step(a, r)
        r1, o1, f1 = host.observe()
        _, o2, _ = ctl.env.observe()
        assert np.array_equal(r1, ctl.rew.cpu().numpy()) and np.array_equal(f1, ctl.first.cpu().numpy()), f"step {t}"
        assert np.array_equal(o1["rgb"], o2["rgb"].cpu().numpy()), f"step {t}: rgb"
    host.close()
    ctl.env.close()
