"""Device-resident steps captured in CUDA graphs (torch.cuda.graph) and replayed.

A graph changes no input of the outputs, so every case runs in lockstep, byte for byte, against an eager handle: the
oracle's record of an existing test replayed through the library (key=..., as test_gpu_launch_shapes.py does), or an
eager device-resident handle on the same inputs where the existing suite already pins the eager path at that size.
Covered: one-step and 8-step graphs, forced launch shapes (16 auxiliary streams, shared ticket slots), 65 536 envs in
the natural 8 chunks, level choice refilled by torch inside the graph, the consumer epilogue's device-resident ring
position, and the calls that refuse to run inside a capture."""
import numpy as np
import pytest

from oracle.record import STANDIN_PACK, oracle_env
from oracle.ref_env import mt19937_actions

pytestmark = pytest.mark.gpu
ALL16 = "bigfish,bossfight,caveflyer,chaser,climber,coinrun,dodgeball,fruitbot,heist,jumper,leaper,maze,miner,ninja,plunder,starpilot"
KW = dict(num_levels=200, start_level=0, rand_seed=0)
HOST_BUFFERS = "test_gpu_parity.py::test_libenv_host_buffers_bit_exact"
COINRUN_HARD_64 = HOST_BUFFERS + "[coinrun-hard-64-1000]#0"
SIXTEEN_64 = "test_gpu_parity.py::test_sixteen_game_list_bit_exact#0"
SMOKE = "smoke#0"   # the record __graft_entry__.smoke() replays: coinrun easy, 16 envs, 48 steps


def _env(n, name, **kw):
    from procgen_b200 import ProcgenGym3Env

    return ProcgenGym3Env(n, name, resource_root=STANDIN_PACK, **kw)


def _matches_record(t, ref, rew, rgb, first, info):
    """Outputs (torch tensors) of step t equal the record replayed by `ref` (oracle_env)."""
    r, o, f = ref.observe()
    assert np.array_equal(rew.cpu().numpy(), r), f"step {t}: rew differs at envs {np.nonzero(rew.cpu().numpy() != r)[0][:8]}"
    assert np.array_equal(first.cpu().numpy().astype(bool), f.astype(bool)), f"step {t}: first"
    got = rgb.cpu().numpy()
    if not np.array_equal(got, o["rgb"]):
        bad = np.nonzero((got != o["rgb"]).reshape(got.shape[0], -1).any(1))[0]
        raise AssertionError(f"step {t}: rgb differs in envs {bad[:8]}")
    for k, v in ref.info.items():
        assert np.array_equal(info[k].cpu().numpy(), v), f"step {t}: info[{k}]"


def _outputs(env):
    rew, ob, first = env.observe()
    return rew, ob["rgb"], first, env.get_info_tensors()


def _capture(fn):
    import torch

    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        fn()
    return g


# ------------------------------------------------------------------ against the oracle's records
@pytest.mark.parametrize("name,mode,n,steps,chunks,serialize,key", [
    ("coinrun", "hard", 64, 1000, 0, False, COINRUN_HARD_64),
    (ALL16, "hard", 64, 500, 5, False, SIXTEEN_64),   # 80 launches a step over the 16 auxiliary streams, ticket slots shared
    ("bossfight", "hard", 32, 800, 7, False, HOST_BUFFERS + "[bossfight-hard-32-800]#0"),
    ("jumper", "hard", 32, 600, 5, False, HOST_BUFFERS + "[jumper-hard-32-600]#0"),
])
def test_one_step_graph_against_record(product_lib, name, mode, n, steps, chunks, serialize, key):
    """One captured step, replayed every step with the step's actions copied into the graph's action buffer."""
    import torch

    env = _env(n, name, distribution_mode=mode, **KW)
    if chunks:
        env.set_launch_shape(chunks, serialize)
    ref = oracle_env(n, name, product_lib, key=key, distribution_mode=mode, **KW)
    acts = torch.as_tensor(mt19937_actions(0, n, steps), device="cuda")
    a = torch.zeros(n, dtype=torch.int32, device="cuda")
    _matches_record(-1, ref, *_outputs(env))
    launches = env.kernel_launches()
    g = _capture(lambda: env.act(a))
    per_step = env.kernel_launches() - launches
    games = len(name.split(","))
    assert per_step == 3 * games * min(max(chunks, 1), n // games), "a captured step issues the eager step's launches (empty chunks launch nothing)"
    for t in range(steps):
        a.copy_(acts[t])
        g.replay()
        ref.act(acts[t].cpu().numpy())
        _matches_record(t, ref, *_outputs(env))
    assert env.kernel_launches() - launches == per_step, "replays are not launches issued"
    assert env.errors() == 0
    ref.close()
    env.close()


def test_eight_step_graph_against_record(product_lib):
    """Eight captured steps reading a static [8, N] action buffer, each step's outputs copied into static buffers
    inside the graph."""
    import torch

    n, steps, w = 64, 1000, 8
    env = _env(n, "coinrun", distribution_mode="hard", **KW)
    ref = oracle_env(n, "coinrun", product_lib, key=COINRUN_HARD_64, distribution_mode="hard", **KW)
    acts = torch.as_tensor(mt19937_actions(0, n, steps), device="cuda")
    a = torch.zeros((w, n), dtype=torch.int32, device="cuda")
    rew = torch.zeros((w, n), dtype=torch.float32, device="cuda")
    rgb = torch.zeros((w, n, 64, 64, 3), dtype=torch.uint8, device="cuda")
    first = torch.zeros((w, n), dtype=torch.bool, device="cuda")
    info = {k: torch.zeros((w,) + v.shape, dtype=v.dtype, device="cuda") for k, v in env.get_info_tensors().items()}
    _matches_record(-1, ref, *_outputs(env))

    def body():
        for i in range(w):
            env.act(a[i])
            r, o, f, inf = _outputs(env)
            rew[i].copy_(r)
            rgb[i].copy_(o)
            first[i].copy_(f)
            for k in info:
                info[k][i].copy_(inf[k])

    g = _capture(body)
    for t0 in range(0, steps, w):
        a.copy_(acts[t0:t0 + w])
        g.replay()
        for i in range(w):
            ref.act(acts[t0 + i].cpu().numpy())
            _matches_record(t0 + i, ref, rew[i], rgb[i], first[i], {k: v[i] for k, v in info.items()})
    assert env.errors() == 0
    ref.close()
    env.close()


# ------------------------------------------------------------------ at size, against an eager handle
def _assert_same(t, a, b):
    ra, oa, fa, ia = _outputs(a)
    rb, ob, fb, ib = _outputs(b)
    bad = (oa != ob).flatten(1).any(1).nonzero().flatten()
    assert bad.numel() == 0, f"step {t}: rgb differs in {bad.numel()} envs, first {bad[:8].tolist()}"
    assert torch_equal(ra, rb) and torch_equal(fa, fb), f"step {t}: rew / first"
    for k in ia:
        assert torch_equal(ia[k], ib[k]), f"step {t}: info[{k}]"


def torch_equal(x, y):
    import torch

    return bool(torch.equal(x, y))


@pytest.mark.parametrize("name,mode", [("coinrun", "easy"), ("bigfish,coinrun", "hard")])
def test_graph_at_size_matches_eager(product_lib, name, mode):
    """65 536 envs per handle, 8 launch chunks per game: a graph handle against an eager handle, every env."""
    import torch

    n, steps = 65536, 30
    kw = dict(distribution_mode=mode, num_levels=0, start_level=0, rand_seed=0)
    genv, eenv = _env(n, name, **kw), _env(n, name, **kw)
    gen = torch.Generator(device="cuda").manual_seed(11)
    acts = torch.randint(0, 15, (steps, n), device="cuda", dtype=torch.int32, generator=gen)
    a = torch.zeros(n, dtype=torch.int32, device="cuda")
    g = _capture(lambda: genv.act(a))
    _assert_same(-1, genv, eenv)
    for t in range(steps):
        a.copy_(acts[t])
        g.replay()
        eenv.act(acts[t])
        _assert_same(t, genv, eenv)
    assert genv.errors() == 0 and eenv.errors() == 0
    genv.close()
    eenv.close()


# ------------------------------------------------------------------ level choice
def test_level_choice_refilled_inside_graph(product_lib):
    """torch refills the consumed entries of next_level_seeds() inside the graph every step (for a seeded half of
    the envs, from a buffer rewritten before each replay); an eager handle gets the same writes."""
    import torch

    n, steps = 256, 200
    kw = dict(distribution_mode="hard", num_levels=0, start_level=0, rand_seed=3)
    genv, eenv = _env(n, "coinrun", **kw), _env(n, "coinrun", **kw)
    for env in (genv, eenv):
        env.set_launch_shape(3)
    gen = torch.Generator(device="cuda").manual_seed(5)
    acts = torch.randint(0, 15, (steps, n), device="cuda", dtype=torch.int32, generator=gen)
    acts[torch.rand((steps, n), device="cuda", generator=gen) < 1 / 16] = -1
    fresh_all = torch.randint(0, 2 ** 31 - 1, (steps, n), device="cuda", dtype=torch.int32, generator=gen)
    subset = torch.rand(n, device="cuda", generator=gen) < 0.5
    gseeds, eseeds = genv.next_level_seeds(), eenv.next_level_seeds()
    a = torch.zeros(n, dtype=torch.int32, device="cuda")
    fresh = torch.zeros(n, dtype=torch.int32, device="cuda")

    def refill(seeds, f):
        seeds.copy_(torch.where(subset & (seeds < 0), f, seeds))

    def body():
        refill(gseeds, fresh)
        genv.act(a)

    g = _capture(body)
    taken = 0
    for t in range(steps):
        a.copy_(acts[t])
        fresh.copy_(fresh_all[t])
        g.replay()
        refill(eseeds, fresh_all[t])
        pending = eseeds.clone()
        eenv.act(acts[t])
        _assert_same(t, genv, eenv)
        assert torch.equal(gseeds, eseeds), f"step {t}: override arrays differ"
        took = eenv.observe()[2] & (pending >= 0)
        taken += int(took.sum())
        assert torch.equal(eenv.get_info_tensors()["level_seed"][took], pending[took]), f"step {t}: an override was not played"
    assert taken > n
    assert genv.errors() == 0 and eenv.errors() == 0
    genv.close()
    eenv.close()


def test_graph_captured_before_level_choice_never_reads_it(product_lib):
    """A graph captured before next_level_seeds() was first requested steps without level choice: replays leave
    the array alone and play the levels an untouched handle plays. An eager step of the same handle takes them."""
    import torch

    n, steps = 64, 40
    kw = dict(distribution_mode="easy", num_levels=0, start_level=0, rand_seed=1)
    genv, ctl = _env(n, "coinrun", **kw), _env(n, "coinrun", **kw)
    a = torch.zeros(n, dtype=torch.int32, device="cuda")
    g = _capture(lambda: genv.act(a))
    seeds = genv.next_level_seeds()
    want = torch.arange(1000, 1000 + n, device="cuda", dtype=torch.int32)
    seeds.copy_(want)
    gen = torch.Generator(device="cuda").manual_seed(2)
    for t in range(steps):
        acts = torch.randint(0, 15, (n,), device="cuda", dtype=torch.int32, generator=gen)
        acts[t % n] = -1   # a reset every step
        a.copy_(acts)
        g.replay()
        ctl.act(acts)
        _assert_same(t, genv, ctl)
    assert torch.equal(seeds, want), "a graph captured before the array existed consumed overrides"
    genv.act(torch.full((n,), -1, device="cuda", dtype=torch.int32))
    assert torch.equal(genv.get_info_tensors()["level_seed"], want), "the eager step did not play the overrides"
    assert bool((seeds == -1).all())
    assert genv.errors() == 0 and ctl.errors() == 0
    genv.close()
    ctl.close()


# ------------------------------------------------------------------ consumer epilogue
def _stack_via_slot(env, k):
    import torch

    s = env.consumer_slot_tensor().to(torch.int64)
    if k == 1:
        return env.consumer_ring()[:, 0]
    idx = s + 1 + torch.arange(k, device="cuda")
    return env.consumer_ring().index_select(1, idx).reshape(env.num, 3 * k, 64, 64)


@pytest.mark.parametrize("dtype_name", ["float16", "bfloat16"])
@pytest.mark.parametrize("k", [1, 4, 16])
def test_consumer_ring_position_on_device(product_lib, dtype_name, k):
    """Replays (37 of them: not a multiple of k), eager steps of the same handle in between, and set_state between
    replays. The stack read through consumer_slot_tensor() equals the eager handle's consumer_observation() and the
    torch-ops restatement of the frames after every step."""
    import torch

    dtype = getattr(torch, dtype_name)
    n, steps = 64, 60
    kw = dict(distribution_mode="easy", num_levels=0, start_level=0, rand_seed=2)
    genv, eenv = _env(n, "coinrun", **kw), _env(n, "coinrun", **kw)
    for env in (genv, eenv):
        env.set_launch_shape(3)   # the ring must move once per step, not once per launch
        env.enable_consumer_output(dtype=dtype, frames=k)
    gen = torch.Generator(device="cuda").manual_seed(7)
    acts = torch.randint(0, 15, (steps, n), device="cuda", dtype=torch.int32, generator=gen)
    a = torch.zeros(n, dtype=torch.int32, device="cuda")
    g = _capture(lambda: genv.act(a))

    def planes(rgb):
        return (rgb.permute(0, 3, 1, 2).to(torch.float32) / 255.0).to(dtype)

    stack = [torch.zeros((n, 3, 64, 64), dtype=dtype, device="cuda") for _ in range(k - 1)] + [planes(eenv.observe()[1]["rgb"])]
    replays = 0
    saved = None
    for t in range(steps):
        if t == 10:
            saved = eenv.get_state()
        if t == 30:
            genv.set_state(saved)
            eenv.set_state(saved)
            _assert_same("after set_state", genv, eenv)
            _, ob, first = eenv.observe()
            stack[-1] = planes(ob["rgb"])   # the restored frame replaces the newest; a restored episode start zeroes the rest
            if k > 1 and bool(first.any()):
                for old in stack[:-1]:
                    old[first] = 0
            assert torch.equal(_stack_via_slot(genv, k), eenv.consumer_observation()), "after set_state"
        if t % 7 == 3:
            genv.act(acts[t])   # an eager step between replays
        else:
            a.copy_(acts[t])
            g.replay()
            replays += 1
        eenv.act(acts[t])
        _assert_same(t, genv, eenv)
        rew, ob, first = eenv.observe()
        stack = stack[1:] + [planes(ob["rgb"])]
        if k > 1 and bool(first.any()):
            for old in stack[:-1]:
                old[first] = 0
        want = torch.cat(stack, dim=1)
        got = _stack_via_slot(genv, k)
        assert torch.equal(eenv.consumer_observation(), want), f"step {t}: eager handle"
        assert torch.equal(got, want), f"step {t}: graph handle's stack read through consumer_slot_tensor()"
        assert torch.equal(genv.consumer_observation(), want), f"step {t}: graph handle's consumer_observation()"
        stack = [x.clone() for x in stack]
    assert replays % k != 0 or k == 1
    if k > 1:
        assert int(genv.consumer_slot_tensor().item()) == steps % k == int(eenv.consumer_slot_tensor().item())
    assert genv.errors() == 0 and eenv.errors() == 0
    genv.close()
    eenv.close()


# ------------------------------------------------------------------ guard rails
def test_refused_calls_inside_capture(product_lib):
    """Every call that waits for the GPU or allocates raises inside torch.cuda.graph and names itself; the handle
    then still steps eagerly, bit-exact against its record, with no error bits."""
    import torch

    n, steps = 16, 48
    kw = dict(distribution_mode="easy", **KW)
    env = _env(n, "coinrun", **kw)
    host = _env(n, "coinrun", host_buffers=True, **kw)
    ref = oracle_env(n, "coinrun", product_lib, key=SMOKE, **kw)
    blobs = env.get_state()
    a = torch.zeros(n, dtype=torch.int32, device="cuda")
    refused = [
        ("get_state", lambda: env.get_state()),
        ("set_state", lambda: env.set_state(blobs)),
        ("errors", lambda: env.errors()),
        ("get_info", lambda: env.get_info()),
        ("enable_consumer_output", lambda: env.enable_consumer_output(torch.float16, 4)),
        ("next_level_seeds", lambda: env.next_level_seeds()),
        ("set_launch_shape", lambda: env.set_launch_shape(2)),
        ("kernel_timing_begin", lambda: env.kernel_timing_begin(8)),
        ("kernel_timing_end", lambda: env.kernel_timing_end()),
        ("enable_peer_gather", lambda: env.enable_peer_gather()),
        ("sync", lambda: env.sync()),
        ("CUDA tensor", lambda: env.act(np.zeros(n, np.int32))),
        ("host_buffers", lambda: host.act(np.zeros(n, np.int32))),
    ]
    for what, call in refused:
        g = torch.cuda.CUDAGraph()
        with pytest.raises(RuntimeError, match=what):
            with torch.cuda.graph(g):
                call()
    acts = mt19937_actions(0, n, steps)
    _matches_record(-1, ref, *_outputs(env))
    for t in range(steps):
        env.act(torch.as_tensor(acts[t], device="cuda"))
        ref.act(acts[t])
        _matches_record(t, ref, *_outputs(env))
    assert env.errors() == 0
    assert env._next_level_seeds is None and getattr(env, "_consumer", None) is None
    ref.close()
    host.close()
    env.close()
