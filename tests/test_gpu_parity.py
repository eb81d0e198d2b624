"""GPU parity tests proper: the CUDA path, called through the C ABI, against the oracle on the same
seeded inputs — bit-exact for rew / first / info AND rgb (the oracle's raster restatement and the
device rasteriser implement the same integer rules, so the tolerance is 0). Both run on the stand-in
asset pack, and the oracle's side is its recorded outputs (oracle/record.py), so the tests need neither
the reference's art nor the oracle library."""
import hashlib
import os

import numpy as np
import pytest

from helpers import make_checked_pair, run_lockstep
from oracle.record import STANDIN_PACK, oracle_env

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


@pytest.mark.parametrize("name,mode,n,steps", [
    ("coinrun", "easy", 64, 1000),   # BASELINE.json configs[0]
    ("coinrun", "hard", 64, 1000),
    ("bigfish", "hard", 64, 1000),   # configs[2] game, small N
    ("bigfish", "easy", 32, 600),
    ("maze", "hard", 64, 800),       # configs[3] games, small N
    ("maze", "easy", 32, 500),
    ("heist", "hard", 64, 800),      # configs[3]; exercises the rotated-sprite raster paths
    ("heist", "easy", 32, 500),
    ("miner", "hard", 32, 600),
    ("leaper", "hard", 32, 600),
    ("plunder", "hard", 32, 800),
    ("chaser", "hard", 32, 600),
    ("climber", "hard", 32, 600),
    ("ninja", "hard", 32, 800),
    ("fruitbot", "hard", 32, 600),
    ("caveflyer", "hard", 32, 600),
    ("bossfight", "hard", 32, 800),
    ("dodgeball", "hard", 32, 600),
    ("dodgeball", "memory", 16, 400),
    ("starpilot", "hard", 32, 800),
    ("starpilot", "extreme", 16, 400),
    ("jumper", "hard", 32, 600),
    ("jumper", "easy", 32, 600),
])
def test_libenv_host_buffers_bit_exact(product_lib, name, mode, n, steps):
    ref, dut = make_checked_pair(product_lib, n, name, distribution_mode=mode, num_levels=200, start_level=0, rand_seed=0)
    run_lockstep(ref, dut, steps)
    ref.close()
    dut.close()


@pytest.mark.parametrize("name", ["coinrun", "bossfight", "chaser", "starpilot", "jumper", "plunder", "heist", "leaper"])
def test_state_blobs_byte_identical_and_portable(product_lib, name):
    from helpers import run_state_roundtrip
    from oracle.ref_env import RefVecEnv

    kw = dict(distribution_mode="hard", num_levels=200, start_level=0)
    run_state_roundtrip(lambda seed: oracle_env(8, name, product_lib, rand_seed=seed, **kw),
                        lambda seed: RefVecEnv(8, name, rand_seed=seed, lib_path=product_lib, resource_root=STANDIN_PACK, **kw),
                        8, 150)


def test_python_api_state_roundtrip(product_lib):
    """ProcgenGym3Env.get_state / set_state (env.py:140-153): restoring a snapshot replays the same frames."""
    import torch

    from procgen_b200 import ProcgenGym3Env

    env = ProcgenGym3Env(16, "coinrun", distribution_mode="hard", num_levels=0, start_level=0, rand_seed=7)
    gen = torch.Generator(device="cuda").manual_seed(3)
    acts = torch.randint(0, 15, (40, 16), device="cuda", dtype=torch.int32, generator=gen)
    for t in range(10):
        env.act(acts[t])
        env.observe()
    states = env.callmethod("get_state")
    frames = []
    for t in range(10, 40):
        env.act(acts[t])
        frames.append(env.observe()[1]["rgb"].clone())
    env.callmethod("set_state", states)
    for t in range(10, 40):
        env.act(acts[t])
        assert torch.equal(env.observe()[1]["rgb"], frames[t - 10])
    assert env.errors() == 0
    env.close()


def test_sixteen_game_list_bit_exact(product_lib):
    """BASELINE.json configs[4] shape on one GPU: env n plays game n % 16."""
    names = "bigfish,bossfight,caveflyer,chaser,climber,coinrun,dodgeball,fruitbot,heist,jumper,leaper,maze,miner,ninja,plunder,starpilot"
    ref, dut = make_checked_pair(product_lib, 64, names, distribution_mode="hard", num_levels=200, start_level=0, rand_seed=0)
    run_lockstep(ref, dut, 500)
    ref.close()
    dut.close()


@pytest.mark.parametrize("fixture", sorted(f for f in os.listdir(GOLDEN) if f.endswith(".npz")))
def test_device_api_reproduces_golden(product_lib, fixture):
    """The device-resident API on the golden fixtures' inputs: rew / first / level_seed equal the fixture (the
    game logic reads only the images' sizes, which the stand-in pack shares with the reference's art), rgb
    equals the oracle's on the stand-in pack."""
    import torch

    from procgen_b200 import ProcgenGym3Env

    g = np.load(os.path.join(GOLDEN, fixture), allow_pickle=False)
    kw = dict(distribution_mode=str(g["mode"]), num_levels=int(g["num_levels"]), start_level=0, rand_seed=int(g["rand_seed"]))
    env = ProcgenGym3Env(int(g["num"]), str(g["env_name"]), resource_root=STANDIN_PACK, **kw)
    ref = oracle_env(int(g["num"]), str(g["env_name"]), product_lib, **kw)
    ref.observe()
    acts = g["actions"]
    for t in range(acts.shape[0]):
        env.act(torch.as_tensor(acts[t], device="cuda"))
        ref.act(acts[t])
        rew, ob, first = env.observe()
        assert np.array_equal(rew.cpu().numpy(), g["rew"][t])
        assert np.array_equal(first.cpu().numpy(), g["first"][t].astype(bool))
        info = env.get_info_tensors()
        assert np.array_equal(info["level_seed"].cpu().numpy(), g["level_seed"][t])
        assert np.array_equal(ob["rgb"].cpu().numpy(), ref.observe()[1]["rgb"]), f"step {t}: rgb"
    assert env.errors() == 0
    env.close()
    ref.close()


ALL16 = "bigfish,bossfight,caveflyer,chaser,climber,coinrun,dodgeball,fruitbot,heist,jumper,leaper,maze,miner,ninja,plunder,starpilot"


@pytest.mark.parametrize("name,mode,n_big,steps", [
    ("coinrun", "easy", 65536, 60),    # BASELINE configs[1]
    ("bigfish", "hard", 65536, 40),    # configs[2]
    ("maze", "hard", 32768, 40),       # configs[3]
    ("heist", "hard", 32768, 40),      # configs[3]
    (ALL16, "hard", 32768, 40),        # configs[4], one GPU's share
    ("bossfight", "hard", 16384, 60),  # hundreds of entities per env: the parallel list compaction under load
    ("jumper", "hard", 16384, 40),     # warp-parallel level generation under load
])
def test_full_size_properties(product_lib, name, mode, n_big, steps):
    """Benchmark-size runs: size-independent properties.
    (a) prefix property: envs [0,64) of the big run == the 64-env oracle run (per-env independence +
        sequential seed chain); (b) run-to-run determinism via a checksum of all observations;
    (c) no env latched an error bit."""
    import torch

    from oracle.ref_env import mt19937_actions
    from procgen_b200 import ProcgenGym3Env

    n_small = 64
    kw = dict(distribution_mode=mode, num_levels=0, start_level=0, rand_seed=0)
    acts_small = mt19937_actions(7, n_small, steps)
    gen = torch.Generator(device="cuda").manual_seed(0)
    acts_big = torch.randint(0, 15, (steps, n_big), device="cuda", dtype=torch.int32, generator=gen)
    acts_big[:, :n_small] = torch.as_tensor(acts_small, device="cuda")

    def run():
        env = ProcgenGym3Env(n_big, name, resource_root=STANDIN_PACK, **kw)
        digest = hashlib.sha256()
        heads = []
        for t in range(steps):
            env.act(acts_big[t])
            rew, ob, first = env.observe()
            heads.append((rew[:n_small].cpu().numpy().copy(), ob["rgb"][:n_small].cpu().numpy().copy(),
                          first[:n_small].cpu().numpy().copy()))
            if t % 10 == 9:
                digest.update(ob["rgb"].cpu().numpy().tobytes())
                digest.update(rew.cpu().numpy().tobytes())
        assert env.errors() == 0
        env.close()
        return digest.hexdigest(), heads

    d1, heads = run()
    d2, _ = run()
    assert d1 == d2
    ref = oracle_env(n_small, name, product_lib, **kw)
    ref.observe()
    for t in range(steps):
        ref.act(acts_small[t])
        rew, ob, first = ref.observe()
        assert np.array_equal(heads[t][0], rew), f"step {t}"
        assert np.array_equal(heads[t][1], ob["rgb"]), f"step {t}"
        assert np.array_equal(heads[t][2], first.astype(bool)), f"step {t}"
    ref.close()


# ------------------------------------------------------------------ round 2: holes named by the review
OTHER_MODES = [
    ("maze", "memory", 8, 300), ("heist", "memory", 8, 300), ("miner", "memory", 8, 300), ("caveflyer", "memory", 8, 300),
    ("jumper", "memory", 8, 300), ("leaper", "extreme", 8, 300), ("chaser", "extreme", 8, 300), ("dodgeball", "extreme", 8, 300),
    ("ninja", "easy", 16, 300), ("fruitbot", "easy", 16, 300), ("bossfight", "easy", 8, 300), ("climber", "easy", 16, 300),
    ("miner", "easy", 16, 300), ("plunder", "easy", 16, 300), ("caveflyer", "easy", 16, 300), ("leaper", "easy", 16, 300),
    ("chaser", "easy", 16, 300), ("dodgeball", "easy", 16, 300), ("starpilot", "easy", 16, 300),
]


@pytest.mark.parametrize("name,mode,n,steps", OTHER_MODES)
def test_remaining_distribution_modes_bit_exact(product_lib, name, mode, n, steps):
    """Every distribution mode each game accepts (game.cpp:56-66) that the main list does not already run."""
    ref, dut = make_checked_pair(product_lib, n, name, distribution_mode=mode, num_levels=200, start_level=0, rand_seed=0)
    run_lockstep(ref, dut, steps)
    ref.close()
    dut.close()


@pytest.mark.parametrize("name,extra", [
    ("coinrun", dict(restrict_themes=True)),
    ("coinrun", dict(use_backgrounds=False)),
    ("heist", dict(center_agent=False)),
    ("maze", dict(use_sequential_levels=True, num_levels=3)),
    ("plunder", dict(restrict_themes=True, use_backgrounds=False)),
    ("coinrun", dict(use_monochrome_assets=True, use_backgrounds=False, restrict_themes=True)),
    ("chaser", dict(use_monochrome_assets=True, use_backgrounds=False)),
    ("ninja", dict(paint_vel_info=True)),
    ("jumper", dict(paint_vel_info=True, use_monochrome_assets=True)),
    ("fruitbot", dict(use_backgrounds=False, restrict_themes=True)),
    ("starpilot", dict(use_backgrounds=False)),
])
def test_non_default_options_bit_exact(product_lib, name, extra):
    kw = dict(distribution_mode="hard", num_levels=200, start_level=0, rand_seed=0)
    kw.update(extra)
    ref, dut = make_checked_pair(product_lib, 8, name, **kw)
    run_lockstep(ref, dut, 250)
    ref.close()
    dut.close()


@pytest.mark.parametrize("name", ["bigfish", "caveflyer", "climber", "dodgeball", "fruitbot", "maze", "miner", "ninja"])
def test_state_blobs_remaining_games(product_lib, name):
    """With test_state_blobs_byte_identical_and_portable: all 16 games' wire format on the GPU."""
    from helpers import run_state_roundtrip
    from oracle.ref_env import RefVecEnv

    kw = dict(distribution_mode="hard", num_levels=200, start_level=0)
    run_state_roundtrip(lambda seed: oracle_env(8, name, product_lib, rand_seed=seed, **kw),
                        lambda seed: RefVecEnv(8, name, rand_seed=seed, lib_path=product_lib, resource_root=STANDIN_PACK, **kw),
                        8, 120)


@pytest.mark.parametrize("name,mode,n_big,warm,steps", [
    ("coinrun", "easy", 65536, 40, 200),   # BASELINE configs[1]
    ("maze", "hard", 32768, 30, 200),      # configs[3]
    ("bigfish", "hard", 65536, 30, 150),   # configs[2]
    (ALL16, "hard", 32768, 30, 150),       # configs[4], one GPU's share
    ("bigfish,coinrun", "hard", 65536, 30, 150),  # a joint list in 8 chunks per game: env_first = g + lo * G
])
def test_mid_array_envs_match_oracle(product_lib, name, mode, n_big, warm, steps):
    """Benchmark-size run, envs picked from EVERY launch chunk (not just the first 64): their state is
    exported through get_state after `warm` steps, loaded into a 64-env oracle, and both are stepped
    with the same actions — rgb / rew / first every step, state blobs at the end."""
    import ctypes as C

    import torch

    from oracle.ref_env import MAX_STATE_SIZE
    from procgen_b200 import ProcgenGym3Env

    n_pick = 64
    n_games = len(name.split(","))
    rs = np.random.RandomState(11)
    # pick j of the oracle plays game j % n_games, so the big env index must be congruent to it; one
    # pick from each of 64 equal slices of the array = every stream chunk is covered several times
    picks = []
    for j in range(n_pick):
        lo, hi = j * (n_big // n_pick), (j + 1) * (n_big // n_pick)
        e = int(rs.randint(lo, hi))
        e = e - (e % n_games) + (j % n_games)
        if e >= hi:
            e -= n_games
        picks.append(e)
    picks = np.array(picks)
    kw = dict(distribution_mode=mode, num_levels=0, start_level=0)
    env = ProcgenGym3Env(n_big, name, rand_seed=0, resource_root=STANDIN_PACK, **kw)
    gen = torch.Generator(device="cuda").manual_seed(5)
    acts = torch.randint(0, 15, (warm + steps, n_big), device="cuda", dtype=torch.int32, generator=gen)
    for t in range(warm):
        env.act(acts[t])
    env.observe()
    buf = C.create_string_buffer(MAX_STATE_SIZE)
    ref = oracle_env(n_pick, name, product_lib, rand_seed=99, **kw)
    for j, e in enumerate(picks):
        nbytes = int(env._lib.get_state(env._h, int(e), buf, MAX_STATE_SIZE))
        ref.set_state(j, bytes(buf.raw[:nbytes]))
    pick_t = torch.as_tensor(picks, device="cuda")
    r0, o0, f0 = ref.observe()
    assert np.array_equal(env.observe()[1]["rgb"][pick_t].cpu().numpy(), o0["rgb"]), "frame after set_state"
    for t in range(warm, warm + steps):
        env.act(acts[t])
        ref.act(acts[t][pick_t].cpu().numpy())
        rew, ob, first = env.observe()
        r, o, f = ref.observe()
        assert np.array_equal(rew[pick_t].cpu().numpy(), r), f"step {t}: rew"
        assert np.array_equal(first[pick_t].cpu().numpy(), f.astype(bool)), f"step {t}: first"
        d = ob["rgb"][pick_t].cpu().numpy()
        assert np.array_equal(d, o["rgb"]), f"step {t}: rgb differs for picks {np.nonzero((d != o['rgb']).reshape(n_pick, -1).any(1))[0][:8]}"
    for j, e in enumerate(picks[::8]):
        nbytes = int(env._lib.get_state(env._h, int(e), buf, MAX_STATE_SIZE))
        assert bytes(buf.raw[:nbytes]) == ref.get_state(j * 8), f"state blob of env {e}"
    assert env.errors() == 0
    env.close()
    ref.close()


@pytest.mark.parametrize("name", ["bossfight", "caveflyer", "ninja", "starpilot"])
def test_long_horizon_trig_games(product_lib, name):
    """10 000 steps (the reference's own state_test horizon, state_test.py:71-124) of the games whose
    logic calls sin / cos / atan2 / pow: CUDA's double-precision libm is <= 2 ulp against glibc's < 1,
    so a difference would need a result within ~1e-16 of a rounding boundary — this is the watch for it."""
    ref, dut = make_checked_pair(product_lib, 8, name, distribution_mode="hard", num_levels=0, start_level=0, rand_seed=3)
    run_lockstep(ref, dut, 10000, seed=1)
    ref.close()
    dut.close()


def test_unsnapped_target_rect_bit_exact(product_lib):
    from helpers import run_snap_off_lockstep

    run_snap_off_lockstep(product_lib, checked=True)


def test_baselines_vecenv_and_gym_wrappers(product_lib):
    """ProcgenEnv / ToBaselinesVecEnv (env.py:249-265) and the procgen-<name>-v0 gym interface
    (gym_registration.py:6-34): same reset/step protocol, same numbers as the oracle."""
    from oracle.ref_env import mt19937_actions
    import procgen_b200

    kw = dict(distribution_mode="easy", num_levels=50, start_level=0, rand_seed=4)
    venv = procgen_b200.ProcgenEnv(num_envs=8, env_name="coinrun", resource_root=STANDIN_PACK, **kw)
    ref = oracle_env(8, "coinrun", product_lib, **kw)
    assert venv.num_envs == 8 and venv.observation_space["rgb"].shape == (64, 64, 3) and venv.action_space.n == 15
    ob = venv.reset()
    assert np.array_equal(ob["rgb"], ref.observe()[1]["rgb"])
    acts = mt19937_actions(2, 8, 150)
    for t in range(150):
        ob, rew, done, infos = venv.step(acts[t])
        ref.act(acts[t])
        r, o, f = ref.observe()
        assert np.array_equal(ob["rgb"], o["rgb"]) and np.array_equal(rew, r) and np.array_equal(done, f.astype(bool))
        assert [i["level_seed"] for i in infos] == list(ref.info["level_seed"])
        assert [i["prev_level_complete"] for i in infos] == list(ref.info["prev_level_complete"])
    assert venv.render(mode="rgb_array").shape == (64, 64, 3)
    venv.close()
    ref.close()

    genv = procgen_b200.make("procgen-maze-v0", distribution_mode="easy", num_levels=20, start_level=0, rand_seed=1,
                             resource_root=STANDIN_PACK)
    ref = oracle_env(1, "maze", product_lib, distribution_mode="easy", num_levels=20, start_level=0, rand_seed=1)
    ob = genv.reset()
    assert ob.shape == (64, 64, 3) and np.array_equal(ob, ref.observe()[1]["rgb"][0])
    acts = mt19937_actions(9, 1, 200)
    for t in range(200):
        ob, rew, done, info = genv.step(int(acts[t][0]))
        ref.act(acts[t])
        r, o, f = ref.observe()
        assert np.array_equal(ob, o["rgb"][0]) and rew == float(r[0]) and done == bool(f[0])
        assert info["level_seed"] == int(ref.info["level_seed"][0])
    genv.close()
    ref.close()


@pytest.mark.parametrize("name,frames,dtype_name", [("coinrun", 4, "float16"), ("bigfish", 1, "bfloat16"), ("maze", 3, "bfloat16")])
def test_consumer_epilogue_matches_torch_ops(product_lib, name, frames, dtype_name):
    """SURVEY §8(f)4: the render kernel's second output (rgb / 255 as 16-bit floats, planar CHW, k-frame
    stack with the VecFrameStack reset rule) equals the same thing computed with torch ops on the
    uint8 observation, element for element."""
    import torch

    from procgen_b200 import ProcgenGym3Env

    dtype = getattr(torch, dtype_name)
    n = 256
    env = ProcgenGym3Env(n, name, distribution_mode="easy", num_levels=0, start_level=0, rand_seed=2)
    env.enable_consumer_output(dtype=dtype, frames=frames)

    def to_planes(rgb):
        return (rgb.permute(0, 3, 1, 2).to(torch.float32) / 255.0).to(dtype)

    rew, ob, first = env.observe()
    stack = [torch.zeros((n, 3, 64, 64), dtype=dtype, device="cuda") for _ in range(frames - 1)] + [to_planes(ob["rgb"])]
    assert torch.equal(env.consumer_observation(), torch.cat(stack, dim=1))
    gen = torch.Generator(device="cuda").manual_seed(1)
    resets = 0
    for t in range(300):
        env.act(torch.randint(0, 15, (n,), device="cuda", dtype=torch.int32, generator=gen))
        rew, ob, first = env.observe()
        newest = to_planes(ob["rgb"])
        stack = stack[1:] + [newest]
        if frames > 1 and bool(first.any()):
            for old in stack[:-1]:
                old[first] = 0
        resets += int(first.sum())
        got = env.consumer_observation()
        assert got.shape == (n, 3 * frames, 64, 64)
        assert torch.equal(got, torch.cat(stack, dim=1)), f"step {t}"
        stack = [x.clone() for x in stack]
    assert resets > 0 and env.errors() == 0
    env.close()


@pytest.mark.parametrize("name,mode", [("coinrun", "hard"), ("ninja", "hard"), ("climber", "hard"), ("caveflyer", "hard"), ("caveflyer", "memory"),
                                       ("jumper", "easy"), ("jumper", "hard"), ("jumper", "memory")])
def test_whole_world_view_of_scrolling_games(product_lib, name, mode):
    """center_agent=False (basic-abstract-game.cpp:819-838) for the scrolling games: the full-view kernels."""
    ref, dut = make_checked_pair(product_lib, 8, name, distribution_mode=mode, num_levels=200, start_level=0, rand_seed=0,
                         center_agent=False)
    run_lockstep(ref, dut, 250)
    ref.close()
    dut.close()
