"""Host logic + the device engine's arithmetic, checked WITHOUT a GPU: the CUDA sources are also
built with g++ (-DPG_HOSTSIM: kernels become loops) purely as a debugging harness, and driven in
lockstep with the oracle through the same libenv C ABI. This is not a product path (the package
refuses to load that build, see test_abi.py); the GPU parity tests proper are in test_gpu_parity.py."""
import pytest

from helpers import make_pair, run_lockstep, run_state_roundtrip

CASES = [
    ("coinrun", "easy", 16, 400),
    ("coinrun", "hard", 16, 400),
    ("bigfish", "easy", 16, 500),
    ("bigfish", "hard", 16, 500),
    ("maze", "easy", 16, 300),
    ("maze", "hard", 16, 500),
    ("maze", "memory", 8, 300),
    ("heist", "easy", 16, 400),     # rotated sprites (agent heading, key ring)
    ("heist", "hard", 16, 500),
    ("heist", "memory", 8, 300),
    ("miner", "hard", 16, 400),
    ("miner", "memory", 8, 300),
    ("leaper", "hard", 16, 400),    # tiled finish line, rotated cars/frog
    ("leaper", "extreme", 8, 300),
    ("plunder", "hard", 16, 500),   # HUD overlay bars, bullets (collides_with_entities)
    ("chaser", "hard", 16, 400),    # maze without dead ends, solid-colour orbs
    ("chaser", "extreme", 8, 300),
    ("climber", "hard", 16, 400),   # custom camera (choose_center)
    ("ninja", "hard", 16, 500),     # bombs/explosions, throwing stars (sin/cos), charge bar
    ("ninja", "easy", 16, 300),
    ("fruitbot", "hard", 16, 400),  # vertically tiled background, tiled barriers and doors
    ("fruitbot", "easy", 16, 300),
    ("caveflyer", "hard", 16, 400),  # cave automaton, free rotation (atan2f), lasers
    ("caveflyer", "memory", 8, 300),
    ("bossfight", "hard", 16, 500),  # hundreds of spinning bullets and trails
    ("bossfight", "easy", 8, 300),
    ("dodgeball", "hard", 16, 400),  # room splitting, lava walls tiled along their length
    ("dodgeball", "extreme", 8, 300),
    ("dodgeball", "memory", 8, 300),
    ("starpilot", "hard", 16, 700),  # std::sort tie order, scrolling tiled background, finish line at t=500
    ("starpilot", "extreme", 8, 300),
    ("jumper", "hard", 16, 400),     # maze + cave generators, compass (ellipse, cosmetic line, bar)
    ("jumper", "easy", 16, 300),     # compass disc on a non-integer rect
    ("jumper", "memory", 8, 300),
]


@pytest.mark.parametrize("name,mode,n,steps", CASES)
def test_lockstep_bit_exact(ref_lib, hostsim_lib, name, mode, n, steps):
    ref, dut = make_pair(hostsim_lib, n, name, distribution_mode=mode, num_levels=200, start_level=0, rand_seed=0)
    run_lockstep(ref, dut, steps)
    ref.close()
    dut.close()


@pytest.mark.parametrize("prog", ["stdsort_check", "atan2f_check"])
def test_native_restatements_match_host_libraries(prog, tmp_path):
    """pg_stdsort.cuh against libstdc++'s std::sort (tie order, heapsort fallback) and pg_atan2f
    against libm's atan2f: the oracle links both libraries, the device cannot."""
    import os
    import subprocess

    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    exe = str(tmp_path / prog)
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-ffp-contract=off", "-I", os.path.join(root, "procgen_b200", "csrc"),
                           os.path.join(root, "tests", "native", prog + ".cpp"), "-o", exe])
    out = subprocess.run([exe], capture_output=True, text=True)
    assert out.returncode == 0 and out.stdout.startswith("OK"), out.stdout[-2000:]


ALL_GAMES = "bigfish,bossfight,caveflyer,chaser,climber,coinrun,dodgeball,fruitbot,heist,jumper,leaper,maze,miner,ninja,plunder,starpilot"


def test_sixteen_game_list_bit_exact(ref_lib, hostsim_lib):
    """BASELINE.json configs[4] shape: env n plays game n % 16 (vecgame.cpp:295-310)."""
    ref, dut = make_pair(hostsim_lib, 32, ALL_GAMES, distribution_mode="hard", num_levels=200, start_level=0, rand_seed=0)
    run_lockstep(ref, dut, 300)
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
])
def test_non_default_options_bit_exact(ref_lib, hostsim_lib, name, extra):
    kw = dict(distribution_mode="hard", num_levels=200, start_level=0, rand_seed=0)
    kw.update(extra)
    ref, dut = make_pair(hostsim_lib, 8, name, **kw)
    run_lockstep(ref, dut, 250)
    ref.close()
    dut.close()


@pytest.mark.parametrize("name", ALL_GAMES.split(","))
def test_state_blobs_byte_identical_and_portable(ref_lib, hostsim_lib, name):
    from oracle.ref_env import RefVecEnv, default_pack

    kw = dict(distribution_mode="hard", num_levels=200, start_level=0)
    run_state_roundtrip(lambda seed: RefVecEnv(4, name, rand_seed=seed, **kw),
                        lambda seed: RefVecEnv(4, name, rand_seed=seed, lib_path=hostsim_lib, resource_root=default_pack(), **kw),
                        4, 100)


def test_unrestricted_levels_and_other_seed(ref_lib, hostsim_lib):
    ref, dut = make_pair(hostsim_lib, 8, "coinrun", distribution_mode="hard", num_levels=0, start_level=0, rand_seed=23)
    run_lockstep(ref, dut, 300, seed=5)
    ref.close()
    dut.close()


def test_sharded_seed_chain_matches_unsharded(ref_lib, hostsim_lib):
    """env_index_offset replays the global per-env seed chain (vecgame.cpp:301-314): shard 1 of 2
    equals envs [8,16) of the 16-env reference."""
    import numpy as np

    from oracle.ref_env import RefVecEnv, default_pack, mt19937_actions

    kw = dict(distribution_mode="easy", num_levels=200, start_level=0, rand_seed=0)
    ref = RefVecEnv(16, "coinrun", **kw)
    shard = RefVecEnv(8, "coinrun", lib_path=hostsim_lib, resource_root=default_pack(),
                      extra_options={"env_index_offset": 8, "env_index_total": 16}, **kw)
    acts = mt19937_actions(3, 16, 120)
    for t in range(120):
        ref.act(acts[t])
        shard.act(acts[t][8:])
        r1, o1, f1 = ref.observe()
        r2, o2, f2 = shard.observe()
        assert np.array_equal(r1[8:], r2) and np.array_equal(f1[8:], f2)
        assert np.array_equal(o1["rgb"][8:], o2["rgb"])
        assert np.array_equal(ref.info["level_seed"][8:], shard.info["level_seed"])
    ref.close()
    shard.close()


def test_unsnapped_target_rect_bit_exact(ref_lib, hostsim_lib):
    """snap_target_rect=False (Qt-5-style phase, DESIGN §2): every cell and sprite takes the general blit path."""
    from helpers import run_snap_off_lockstep

    run_snap_off_lockstep(hostsim_lib)


@pytest.mark.parametrize("name", ALL_GAMES.split(","))
def test_restrict_themes_all_games(ref_lib, hostsim_lib, name):
    """restrict_themes masks the theme inside initialize_asset_if_necessary (basic-abstract-game.cpp:86), so
    it changes the aspect ratios game LOGIC reads (match_aspect_ratio / fit_aspect_ratio), not only the
    sprites drawn — every game, because each has its own multi-theme types."""
    ref, dut = make_pair(hostsim_lib, 8, name, distribution_mode="hard", num_levels=200, start_level=0, rand_seed=0,
                         restrict_themes=True)
    run_lockstep(ref, dut, 150)
    ref.close()
    dut.close()


@pytest.mark.parametrize("name,mode", [("coinrun", "hard"), ("coinrun", "easy"), ("ninja", "hard"), ("climber", "hard"),
                                       ("caveflyer", "hard"), ("caveflyer", "memory"), ("jumper", "easy"), ("jumper", "hard"),
                                       ("jumper", "memory")])
def test_whole_world_view_of_scrolling_games(ref_lib, hostsim_lib, name, mode):
    """center_agent=False for the games that otherwise scroll (basic-abstract-game.cpp:819-838): the whole
    world — up to 64 x 64 cells of about one pixel — through the full-view instantiation of the setup /
    render kernels."""
    ref, dut = make_pair(hostsim_lib, 8, name, distribution_mode=mode, num_levels=200, start_level=0, rand_seed=0,
                         center_agent=False)
    run_lockstep(ref, dut, 200)
    ref.close()
    dut.close()


# ---- launch shapes: VecEnv::launch cuts a step into (game, env chunk) launches; at benchmark sizes a
# step has 8 chunks per game. pgb200_set_launch_shape forces the chunk count here, so the chunk index
# arithmetic (env_first = g + lo * G, env_step = G, uneven and empty chunks) runs at oracle sizes.
@pytest.mark.parametrize("name,n,chunks", [
    ("coinrun", 16, 3),        # uneven chunks (5, 5, 6)
    ("coinrun", 16, 16),       # one env per chunk
    ("coinrun", 16, 40),       # 24 empty chunks
    ("coinrun", 13, 4),        # odd n: partial setup / logic blocks in every chunk
    (ALL_GAMES, 32, 5),        # joint list: 2 envs per game in 5 chunks, 3 of them empty
    (ALL_GAMES, 64, 3),        # joint list: 4 envs per game in 3 uneven chunks
    ("caveflyer,heist,starpilot", 21, 3),
])
def test_forced_launch_shapes_bit_exact(ref_lib, hostsim_lib, name, n, chunks):
    ref, dut = make_pair(hostsim_lib, n, name, launch_shape=(chunks, False), distribution_mode="hard", num_levels=200,
                         start_level=0, rand_seed=0)
    run_lockstep(ref, dut, 200)
    ref.close()
    dut.close()


@pytest.mark.parametrize("name,n", [("coinrun", 1), ("coinrun", 3), ("coinrun", 13), ("heist", 5), ("bossfight", 7),
                                    ("caveflyer,heist,starpilot", 21)])
def test_odd_env_counts_bit_exact(ref_lib, hostsim_lib, name, n):
    """Env counts that leave a partial block in every kernel (4 envs per setup block, 2 per logic block)."""
    ref, dut = make_pair(hostsim_lib, n, name, distribution_mode="hard", num_levels=200, start_level=0, rand_seed=0)
    run_lockstep(ref, dut, 300)
    ref.close()
    dut.close()


@pytest.mark.parametrize("name,n,chunks", [(ALL_GAMES, 16, 3), ("caveflyer,heist,starpilot", 9, 2)])
def test_state_blobs_into_joint_list(ref_lib, hostsim_lib, name, n, chunks):
    """set_state into a joint list: env e is game e % G (gi = env_idx % G), re-rendered by a one-env launch;
    the fresh envs the blobs are loaded into step in forced chunks afterwards."""
    from oracle.ref_env import RefVecEnv, default_pack

    kw = dict(distribution_mode="hard", num_levels=200, start_level=0)
    run_state_roundtrip(lambda seed: RefVecEnv(n, name, rand_seed=seed, **kw),
                        lambda seed: RefVecEnv(n, name, rand_seed=seed, lib_path=hostsim_lib, resource_root=default_pack(),
                                               launch_shape=(chunks, False), **kw),
                        n, 100)


def test_set_state_leaves_other_envs_alone(ref_lib, hostsim_lib):
    """Loading one env of a chunk changes that env only: the others go on exactly as in a run without it."""
    import numpy as np

    from oracle.ref_env import RefVecEnv, default_pack, mt19937_actions

    kw = dict(distribution_mode="hard", num_levels=200, start_level=0, rand_seed=0, lib_path=hostsim_lib,
              resource_root=default_pack(), launch_shape=(3, False))
    n, names = 24, "caveflyer,heist,starpilot"
    a, b = RefVecEnv(n, names, **kw), RefVecEnv(n, names, **kw)
    donor = RefVecEnv(n, names, **dict(kw, rand_seed=9))
    acts = mt19937_actions(4, n, 120)
    for t in range(60):
        for env in (a, b, donor):
            env.act(acts[t])
    targets = [1, 11, 22]
    for e in targets:
        b.set_state(e, donor.get_state(e))
    others = np.setdiff1d(np.arange(n), targets)
    for t in range(60, 120):
        for env in (a, b, donor):
            env.act(acts[t])
            env.observe()
        assert np.array_equal(a.rgb[others], b.rgb[others]) and np.array_equal(a.rew[others], b.rew[others]), f"step {t}"
        assert np.array_equal(donor.rgb[targets], b.rgb[targets]) and np.array_equal(donor.first[targets], b.first[targets]), f"step {t}"
    for env in (a, b, donor):
        env.close()


def test_staging_path_with_scattered_observation_slots(ref_lib, hostsim_lib):
    """Observation pointers that are not one contiguous block (reversed env order, every other frame of a
    larger array) take the staging buffer and the per-env scatter."""
    layout = [2 * (12 - 1 - e) for e in range(12)]
    ref, dut = make_pair(hostsim_lib, 12, "maze", launch_shape=(5, False), ob_layout=layout, distribution_mode="hard",
                         num_levels=200, start_level=0, rand_seed=0)
    run_lockstep(ref, dut, 200)
    ref.close()
    dut.close()
