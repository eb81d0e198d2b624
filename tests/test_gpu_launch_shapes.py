"""GPU parity for the launch shapes the vector runtime produces, not just one launch per game.

VecEnv::launch (procgen_b200/csrc/pg_runtime.cu) cuts a step into (game, env chunk) launches: 8 chunks per
game from 4096 * 8 envs per game up, one below. The oracle-sized tests of test_gpu_parity.py therefore run
one launch per game; here pgb200_set_launch_shape forces uneven, one-env and empty chunks, shared ticket
slots (more than 64 launches in a step) and back-to-back launches at oracle sizes, and the runs that do have
natural chunks are compared env for env with the device-resident path (which test_gpu_parity.py pins to the
oracle at those sizes). Also here: odd env counts (partial blocks), the host-buffer observation paths
(per-chunk DMA, staging buffer), set_state into the device, the consumer epilogue beyond one launch, and
several handles and torch streams in one process.

A launch shape is not an input of the oracle's outputs, so a forced-shape rerun of an oracle-compared case
replays that case's record (key=...)."""
import ctypes as C

import numpy as np
import pytest

from helpers import make_checked_pair, run_lockstep, run_state_roundtrip
from oracle.record import STANDIN_PACK, oracle_env
from oracle.ref_env import MAX_STATE_SIZE, RefVecEnv, mt19937_actions

pytestmark = pytest.mark.gpu
ALL16 = "bigfish,bossfight,caveflyer,chaser,climber,coinrun,dodgeball,fruitbot,heist,jumper,leaper,maze,miner,ninja,plunder,starpilot"
THREE = "caveflyer,heist,starpilot"
KW = dict(num_levels=200, start_level=0, rand_seed=0)
HOST_BUFFERS = "test_gpu_parity.py::test_libenv_host_buffers_bit_exact"
COINRUN_HARD_64 = HOST_BUFFERS + "[coinrun-hard-64-1000]#0"
SIXTEEN_64 = "test_gpu_parity.py::test_sixteen_game_list_bit_exact#0"


@pytest.mark.parametrize("name,mode,n,steps,chunks,serialize,key", [
    ("coinrun", "hard", 64, 1000, 3, False, COINRUN_HARD_64),    # uneven chunks (21, 21, 22)
    ("coinrun", "hard", 64, 1000, 8, True, COINRUN_HARD_64),     # the benchmark's chunk count, launches back to back
    ("coinrun", "hard", 64, 1000, 64, False, COINRUN_HARD_64),   # one env per chunk
    ("coinrun", "hard", 64, 1000, 100, False, COINRUN_HARD_64),  # 36 empty chunks
    (ALL16, "hard", 64, 500, 2, False, SIXTEEN_64),
    (ALL16, "hard", 64, 500, 5, False, SIXTEEN_64),               # 80 launches a step: ticket slots shared
    (ALL16, "hard", 64, 500, 5, True, SIXTEEN_64),
    ("bossfight", "hard", 32, 800, 7, False, HOST_BUFFERS + "[bossfight-hard-32-800]#0"),  # entity-heavy
    ("jumper", "hard", 32, 600, 5, False, HOST_BUFFERS + "[jumper-hard-32-600]#0"),        # level generation in the logic kernel
])
def test_forced_chunks_bit_exact(product_lib, name, mode, n, steps, chunks, serialize, key):
    ref, dut = make_checked_pair(product_lib, n, name, key=key, launch_shape=(chunks, serialize), distribution_mode=mode, **KW)
    run_lockstep(ref, dut, steps)
    ref.close()
    dut.close()


@pytest.mark.parametrize("name,n", [("coinrun", 1), ("coinrun", 3), ("coinrun", 13), ("heist", 5), ("bossfight", 7), (THREE, 21)])
def test_odd_env_counts_bit_exact(product_lib, name, n):
    """Env counts that leave a partial block in every kernel (4 envs per setup block, 2 per logic block)."""
    ref, dut = make_checked_pair(product_lib, n, name, distribution_mode="hard", **KW)
    run_lockstep(ref, dut, 300)
    ref.close()
    dut.close()


def test_three_game_list_in_chunks_bit_exact(product_lib):
    ref, dut = make_checked_pair(product_lib, 21, THREE, key=f"test_gpu_launch_shapes.py::test_odd_env_counts_bit_exact[{THREE}-21]#0",
                                 launch_shape=(3, False), distribution_mode="hard", **KW)
    run_lockstep(ref, dut, 300)
    ref.close()
    dut.close()


# ------------------------------------------------------------------ host-buffer observation paths at size
def _assert_host_equals_device(t, rgb, rew, first, info, denv):
    """Outputs of a host-buffer handle (numpy) equal those of the device-resident handle `denv`, every env."""
    import torch

    drew, dob, dfirst = denv.observe()
    assert np.array_equal(rew, drew.cpu().numpy()), f"step {t}: rew differs at envs {np.nonzero(rew != drew.cpu().numpy())[0][:8]}"
    assert np.array_equal(np.asarray(first).astype(bool), dfirst.cpu().numpy()), f"step {t}: first"
    dinfo = denv.get_info_tensors()
    for k in ("prev_level_seed", "prev_level_complete", "level_seed"):
        assert np.array_equal(info[k], dinfo[k].cpu().numpy()), f"step {t}: info[{k}]"
    bad = (torch.as_tensor(rgb).to(dob["rgb"].device) != dob["rgb"]).flatten(1).any(1).nonzero().flatten()
    assert bad.numel() == 0, f"step {t}: rgb differs in {bad.numel()} envs, first {bad[:8].tolist()}"


def test_direct_dma_at_size_matches_device_path(product_lib):
    """65 536 coinrun envs with host buffers, 8 natural chunks: each chunk's observation DMA is queued right
    behind its render kernel into the caller's page-locked array (what bench.py's e2e leg times)."""
    import torch

    from procgen_b200 import ProcgenGym3Env

    n, steps = 65536, 30
    kw = dict(distribution_mode="easy", num_levels=0, start_level=0, rand_seed=0, resource_root=STANDIN_PACK)
    henv = ProcgenGym3Env(n, "coinrun", host_buffers=True, **kw)
    denv = ProcgenGym3Env(n, "coinrun", **kw)
    acts = mt19937_actions(3, n, steps)
    rew, ob, first = henv.observe()
    _assert_host_equals_device(-1, ob["rgb"], rew, first, henv._info, denv)
    for t in range(steps):
        henv.act(acts[t])
        denv.act(torch.as_tensor(acts[t], device="cuda"))
        rew, ob, first = henv.observe()
        _assert_host_equals_device(t, ob["rgb"], rew, first, henv._info, denv)
    assert henv.errors() == 0 and denv.errors() == 0
    henv.close()
    denv.close()


def test_staging_path_at_size_matches_device_path(product_lib):
    """32 768 maze envs through the raw libenv ABI with the observation slots in reversed env order: not one
    contiguous block, so frames go through the staging buffer and the per-env scatter."""
    import torch

    from procgen_b200 import ProcgenGym3Env

    n, steps = 32768, 30
    kw = dict(distribution_mode="hard", num_levels=0, start_level=0, rand_seed=0)
    henv = RefVecEnv(n, "maze", lib_path=product_lib, resource_root=STANDIN_PACK, ob_layout=list(range(n - 1, -1, -1)), **kw)
    denv = ProcgenGym3Env(n, "maze", resource_root=STANDIN_PACK, **kw)
    acts = mt19937_actions(4, n, steps)
    rew, ob, first = henv.observe()
    _assert_host_equals_device(-1, ob["rgb"], rew, first, henv.info, denv)
    for t in range(steps):
        henv.act(acts[t])
        denv.act(torch.as_tensor(acts[t], device="cuda"))
        rew, ob, first = henv.observe()
        _assert_host_equals_device(t, ob["rgb"], rew, first, henv.info, denv)
    assert denv.errors() == 0
    henv.close()
    denv.close()


def test_staging_path_in_chunks_bit_exact(product_lib):
    """The staging path at oracle size: every other frame of a larger array, in reversed order, 5 chunks."""
    ref, dut = make_checked_pair(product_lib, 64, "coinrun", key=COINRUN_HARD_64, launch_shape=(5, False),
                                 ob_layout=[2 * (63 - e) for e in range(64)], distribution_mode="hard", **KW)
    run_lockstep(ref, dut, 1000)
    ref.close()
    dut.close()


# ------------------------------------------------------------------ set_state into the device
def test_state_blobs_into_joint_list(product_lib):
    """run_state_roundtrip on the 16-game list: set_state picks game env_idx % 16 and re-renders that env
    with a one-env launch; the library steps in 3 chunks per game (2 of them empty)."""
    kw = dict(distribution_mode="hard", num_levels=200, start_level=0)
    run_state_roundtrip(lambda seed: oracle_env(32, ALL16, product_lib, rand_seed=seed, **kw),
                        lambda seed: RefVecEnv(32, ALL16, rand_seed=seed, lib_path=product_lib, resource_root=STANDIN_PACK,
                                               launch_shape=(3, False), **kw),
                        32, 100)


def test_oracle_states_into_mid_array_envs(product_lib):
    """The oracle's states loaded into 64 envs spread over all 8 chunks of a 65 536-env handle: those envs
    then follow the oracle, and every other env follows a control handle that was not touched."""
    import torch

    from procgen_b200 import ProcgenGym3Env

    n_big, n_pick, warm, steps = 65536, 64, 20, 60
    kw = dict(distribution_mode="easy", num_levels=0, start_level=0)
    rs = np.random.RandomState(13)
    picks = np.array([int(rs.randint(j * (n_big // n_pick), (j + 1) * (n_big // n_pick))) for j in range(n_pick)])
    ref = oracle_env(n_pick, "coinrun", product_lib, rand_seed=99, **kw)
    oacts = mt19937_actions(6, n_pick, warm)
    ref.observe()
    for t in range(warm):
        ref.act(oacts[t])
        ref.observe()
    blobs = [ref.get_state(j) for j in range(n_pick)]

    env = ProcgenGym3Env(n_big, "coinrun", rand_seed=0, resource_root=STANDIN_PACK, **kw)
    ctl = ProcgenGym3Env(n_big, "coinrun", rand_seed=0, resource_root=STANDIN_PACK, **kw)
    gen = torch.Generator(device="cuda").manual_seed(8)
    acts = torch.randint(0, 15, (warm + steps, n_big), device="cuda", dtype=torch.int32, generator=gen)
    for t in range(warm):
        env.act(acts[t])
        ctl.act(acts[t])
    env.observe()
    for j, e in enumerate(picks):
        env._lib.set_state(env._h, int(e), blobs[j], len(blobs[j]))
    pick_t = torch.as_tensor(picks, device="cuda")
    others = torch.ones(n_big, dtype=torch.bool, device="cuda")
    others[pick_t] = False

    def check(t, r, o, f):
        rew, ob, first = env.observe()
        crew, cob, cfirst = ctl.observe()
        assert np.array_equal(ob["rgb"][pick_t].cpu().numpy(), o["rgb"]), f"step {t}: rgb of the loaded envs"
        assert np.array_equal(rew[pick_t].cpu().numpy(), r) and np.array_equal(first[pick_t].cpu().numpy(), f.astype(bool)), f"step {t}"
        assert torch.equal(ob["rgb"][others], cob["rgb"][others]), f"step {t}: rgb of an env set_state did not address"
        assert torch.equal(rew[others], crew[others]) and torch.equal(first[others], cfirst[others]), f"step {t}"

    check("after set_state", *ref.observe())
    for t in range(warm, warm + steps):
        env.act(acts[t])
        ctl.act(acts[t])
        ref.act(acts[t][pick_t].cpu().numpy())
        check(t, *ref.observe())
    assert env.errors() == 0 and ctl.errors() == 0
    env.close()
    ctl.close()
    ref.close()


def test_set_state_between_act_and_observe_host_buffers(product_lib):
    """Host-buffer mode queues the observation DMA behind the step's render kernels; a set_state after act()
    must make the next observe() return the restored frame, not the one that DMA carried."""
    from procgen_b200 import ProcgenGym3Env

    n = 512
    kw = dict(distribution_mode="easy", num_levels=0, start_level=0, rand_seed=1, resource_root=STANDIN_PACK, host_buffers=True)
    env, ctl = ProcgenGym3Env(n, "coinrun", **kw), ProcgenGym3Env(n, "coinrun", **kw)
    env.set_launch_shape(4)
    acts = mt19937_actions(2, n, 21)
    targets = [0, 130, 257, 511]
    for t in range(21):
        if t == 20:
            env.act(acts[t])
            ctl.act(acts[t])
            for e in targets:
                env._lib.set_state(env._h, e, saved[e], len(saved[e]))
            rew, ob, first = env.observe()
            crew, cob, cfirst = ctl.observe()
            others = np.setdiff1d(np.arange(n), targets)
            assert np.array_equal(ob["rgb"][targets], saved_rgb), "set_state after act: the observed frame is not the restored one"
            assert np.array_equal(rew[targets], saved_rew)
            assert np.array_equal(ob["rgb"][others], cob["rgb"][others]) and np.array_equal(rew[others], crew[others])
            break
        env.act(acts[t])
        ctl.act(acts[t])
        env.observe()
        ctl.observe()
        if t == 10:
            buf = C.create_string_buffer(MAX_STATE_SIZE)
            saved = {}
            for e in targets:
                nbytes = int(env._lib.get_state(env._h, e, buf, MAX_STATE_SIZE))
                saved[e] = bytes(buf.raw[:nbytes])
            saved_rgb = env._rgb[targets].copy()
            saved_rew = env._rew[targets].copy()
    assert not np.array_equal(saved_rgb, ctl._rgb[targets]), "the run is too short to tell restored frames from current ones"
    env.close()
    ctl.close()


# ------------------------------------------------------------------ consumer epilogue beyond one launch
def _consumer_check(env, dtype, frames, steps, gen, seen=None):
    """The consumer output after every step equals the torch-ops restatement (the test_gpu_parity.py one:
    rgb / 255 in fp32, rounded to the 16-bit type, CHW planes, k-frame stack zeroed on episode start)."""
    import torch

    n = env.num

    def to_planes(rgb):
        return (rgb.permute(0, 3, 1, 2).to(torch.float32) / 255.0).to(dtype)

    rew, ob, first = env.observe()
    stack = [torch.zeros((n, 3, 64, 64), dtype=dtype, device="cuda") for _ in range(frames - 1)] + [to_planes(ob["rgb"])]
    assert torch.equal(env.consumer_observation(), torch.cat(stack, dim=1)), "after enable"
    resets = 0
    for t in range(steps):
        env.act(torch.randint(0, 15, (n,), device="cuda", dtype=torch.int32, generator=gen))
        rew, ob, first = env.observe()
        stack = stack[1:] + [to_planes(ob["rgb"])]
        if frames > 1 and bool(first.any()):
            for old in stack[:-1]:
                old[first] = 0
        resets += int(first.sum())
        if seen is not None:
            seen |= torch.bincount(ob["rgb"].flatten(), minlength=256) > 0
        got = env.consumer_observation()
        assert got.shape == (n, 3 * frames, 64, 64)
        assert torch.equal(got, torch.cat(stack, dim=1)), f"step {t}: consumer output differs from the torch-ops restatement"
        stack = [x.clone() for x in stack]
    return resets


@pytest.mark.parametrize("name,mode,n,frames,dtype_name,extra,chunks,steps", [
    (ALL16, "hard", 64, 4, "float16", {}, 0, 150),                      # joint list: env_first = g, env_step = 16
    ("coinrun", "easy", 256, 3, "bfloat16", {}, 5, 200),                # forced chunks
    ("caveflyer", "hard", 64, 2, "float16", dict(center_agent=False), 0, 200),  # whole-world render kernel
    ("bigfish", "easy", 64, 16, "bfloat16", {}, 0, 60),                 # k = 16: a ring of 32 slots
])
def test_consumer_epilogue_launch_shapes(product_lib, name, mode, n, frames, dtype_name, extra, chunks, steps):
    import torch

    from procgen_b200 import ProcgenGym3Env

    dtype = getattr(torch, dtype_name)
    env = ProcgenGym3Env(n, name, distribution_mode=mode, num_levels=0, start_level=0, rand_seed=2, resource_root=STANDIN_PACK, **extra)
    if chunks:
        env.set_launch_shape(chunks)
    env.enable_consumer_output(dtype=dtype, frames=frames)
    seen = torch.zeros(256, dtype=torch.bool, device="cuda")
    resets = _consumer_check(env, dtype, frames, steps, torch.Generator(device="cuda").manual_seed(1), seen)
    assert resets > 0 and env.errors() == 0
    if name == ALL16:
        # every byte value went through the LUT and was compared at least once
        assert bool(seen.all()), f"byte values never compared: {(~seen).nonzero().flatten().tolist()[:16]}"
    env.close()


def test_consumer_epilogue_enabled_mid_run_and_switched(product_lib):
    """Enabled after 50 steps (the current frames become the newest of an empty stack), then re-enabled
    with the other 16-bit type and another k."""
    import torch

    from procgen_b200 import ProcgenGym3Env

    env = ProcgenGym3Env(256, "coinrun", distribution_mode="easy", num_levels=0, start_level=0, rand_seed=4, resource_root=STANDIN_PACK)
    env.set_launch_shape(3)
    gen = torch.Generator(device="cuda").manual_seed(5)
    for t in range(50):
        env.act(torch.randint(0, 15, (256,), device="cuda", dtype=torch.int32, generator=gen))
    env.enable_consumer_output(dtype=torch.float16, frames=4)
    resets = _consumer_check(env, torch.float16, 4, 120, gen)
    env.enable_consumer_output(dtype=torch.bfloat16, frames=2)
    resets += _consumer_check(env, torch.bfloat16, 2, 120, gen)
    assert resets > 0 and env.errors() == 0
    env.close()


# ------------------------------------------------------------------ several handles, torch streams
def _device_step_matches(env, ref, t):
    rew, ob, first = env.observe()
    r, o, f = ref.observe()
    assert np.array_equal(rew.cpu().numpy(), r), f"step {t}: rew"
    assert np.array_equal(first.cpu().numpy(), f.astype(bool)), f"step {t}: first"
    assert np.array_equal(ob["rgb"].cpu().numpy(), o["rgb"]), f"step {t}: rgb"
    info = env.get_info_tensors()
    for k, v in ref.info.items():
        assert np.array_equal(info[k].cpu().numpy(), v), f"step {t}: info[{k}]"


def test_two_handles_interleaved_on_torch_streams(product_lib):
    """A coinrun handle and a 16-game-list handle, both device-resident, stepped in turn: on one torch stream
    for the first half of the list's run, then each on its own stream. The oracle's records replay through
    two host-buffer handles alive beside them."""
    import torch

    from procgen_b200 import ProcgenGym3Env

    kw = dict(distribution_mode="hard", resource_root=STANDIN_PACK, **KW)
    a = ProcgenGym3Env(64, "coinrun", **kw)
    b = ProcgenGym3Env(64, ALL16, **kw)
    ref_a = oracle_env(64, "coinrun", product_lib, key=COINRUN_HARD_64, distribution_mode="hard", **KW)
    ref_b = oracle_env(64, ALL16, product_lib, key=SIXTEEN_64, distribution_mode="hard", **KW)
    acts_a, acts_b = mt19937_actions(0, 64, 1000), mt19937_actions(0, 64, 500)
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    with torch.cuda.stream(s1):
        _device_step_matches(a, ref_a, -1)
        _device_step_matches(b, ref_b, -1)
    for t in range(1000):
        with torch.cuda.stream(s1):
            a.act(torch.as_tensor(acts_a[t], device="cuda"))
            ref_a.act(acts_a[t])
        if t < 500:
            with torch.cuda.stream(s1 if t < 250 else s2):
                b.act(torch.as_tensor(acts_b[t], device="cuda"))
                ref_b.act(acts_b[t])
                _device_step_matches(b, ref_b, t)
        with torch.cuda.stream(s1):
            _device_step_matches(a, ref_a, t)
    assert a.errors() == 0 and b.errors() == 0
    for env in (a, b, ref_a, ref_b):
        env.close()


def test_act_alternating_torch_streams(product_lib):
    """act() on another torch stream every step: the handle follows the caller's current stream."""
    import torch

    from procgen_b200 import ProcgenGym3Env

    kw = dict(distribution_mode="easy", num_levels=200, start_level=0, rand_seed=0)
    env = ProcgenGym3Env(16, "coinrun", resource_root=STANDIN_PACK, **kw)
    ref = oracle_env(16, "coinrun", product_lib, key="smoke#0", **kw)   # the record __graft_entry__.smoke() replays
    acts = mt19937_actions(0, 16, 48)
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    _device_step_matches(env, ref, -1)
    for t in range(48):
        with torch.cuda.stream(streams[t % 2]):
            env.act(torch.as_tensor(acts[t], device="cuda"))
            ref.act(acts[t])
            _device_step_matches(env, ref, t)
    assert env.errors() == 0
    env.close()
    ref.close()
