"""Shared test helpers: lockstep comparison of any libenv-ABI implementation against the oracle."""
import ctypes as C
import os

import numpy as np

from oracle.record import STANDIN_PACK, oracle_env
from oracle.ref_env import RefVecEnv, default_pack, mt19937_actions


def make_pair(lib_path, num, env_name, extra_options=None, launch_shape=None, ob_layout=None, **kw):
    """(the oracle, the library under test); launch_shape and ob_layout apply to the library under test only."""
    ref = RefVecEnv(num, env_name, **kw)
    dut = RefVecEnv(num, env_name, lib_path=lib_path, resource_root=default_pack(), extra_options=extra_options,
                    launch_shape=launch_shape, ob_layout=ob_layout, **kw)
    return ref, dut


def make_checked_pair(lib_path, num, env_name, extra_options=None, launch_shape=None, ob_layout=None, key=None, **kw):
    """(oracle_env: the oracle's recorded outputs, the library under test), both on the stand-in asset pack.
    launch_shape and ob_layout apply to the library under test only; they are not inputs of the outputs, so a
    run that only changes them may replay the record of another test (key)."""
    ref = oracle_env(num, env_name, lib_path, key=key, extra_options=extra_options, **kw)
    dut = RefVecEnv(num, env_name, lib_path=lib_path, resource_root=STANDIN_PACK, extra_options=extra_options,
                    launch_shape=launch_shape, ob_layout=ob_layout, **kw)
    return ref, dut


def lib_array(env, ptr, shape, typestr):
    """An array the library under test hands out for a libenv-ABI env (oracle.ref_env.RefVecEnv), at `ptr` (an
    address or a ctypes pointer): a numpy view in the host debug build, a torch CUDA tensor aliasing device memory
    in the GPU build."""
    env.lib.pgb200_is_device_build.restype = C.c_int
    addr = ptr if isinstance(ptr, int) else C.cast(ptr, C.c_void_p).value
    if not env.lib.pgb200_is_device_build():
        ctype = np.ctypeslib.as_ctypes_type(np.dtype(typestr))
        return np.ctypeslib.as_array(C.cast(addr, C.POINTER(ctype)), shape=shape)
    import torch

    from procgen_b200.env import _CudaArray

    return torch.as_tensor(_CudaArray(addr, shape, typestr), device="cuda")


def write_lib_array(arr, values):
    """Write the whole of a lib_array; a device array is written with torch and synchronised (libenv_act needs the
    writes complete before it is called)."""
    if isinstance(arr, np.ndarray):
        arr[:] = values
        return
    import torch

    arr.copy_(torch.as_tensor(np.asarray(values)).to(arr.device))
    torch.cuda.synchronize()


def read_lib_array(arr):
    """A host copy of a lib_array, once the device's work so far is complete."""
    if isinstance(arr, np.ndarray):
        return arr.copy()
    import torch

    torch.cuda.synchronize()
    return arr.cpu().numpy()


def assert_same_observation(ref, dut, t, rgb_tol=0):
    r1, o1, f1 = ref.observe()
    r2, o2, f2 = dut.observe()
    assert np.array_equal(r1, r2), f"step {t}: rew differs at envs {np.nonzero(r1 != r2)[0][:8]}"
    assert np.array_equal(f1, f2), f"step {t}: first differs at envs {np.nonzero(f1 != f2)[0][:8]}"
    for k in ref.info:
        assert np.array_equal(ref.info[k], dut.info[k]), f"step {t}: info[{k}] differs"
    if rgb_tol == 0:
        if not np.array_equal(o1["rgb"], o2["rgb"]):
            d = np.abs(o1["rgb"].astype(int) - o2["rgb"].astype(int))
            bad = np.nonzero(d.reshape(d.shape[0], -1).sum(1))[0]
            raise AssertionError(f"step {t}: rgb differs in envs {bad[:8]}, {int((d.sum(-1) > 0).sum())} px, max |d| {d.max()}")
    else:
        d = np.abs(o1["rgb"].astype(int) - o2["rgb"].astype(int))
        assert d.max() <= rgb_tol, f"step {t}: rgb max |d| {d.max()} > {rgb_tol}"


def run_lockstep(ref, dut, steps, seed=0, rgb_tol=0):
    acts = mt19937_actions(seed, ref.num, steps)
    assert_same_observation(ref, dut, -1, rgb_tol)
    for t in range(steps):
        ref.act(acts[t])
        dut.act(acts[t])
        assert_same_observation(ref, dut, t, rgb_tol)
    if hasattr(dut.lib, "pgb200_get_errors"):
        import ctypes as C

        dut.lib.pgb200_get_errors.restype = C.c_uint32
        err = dut.lib.pgb200_get_errors(C.c_void_p(dut.h), None)
        assert err == 0, f"device latched error bits {err:#x} (capacity overflow / unsupported feature)"


def run_state_roundtrip(make_ref, make_dut, num, steps, check_every=25):
    """Full-state parity through the reference's own wire format (vecgame.cpp:437-457), following the
    shape of the reference's state_test.py: (1) the blobs of both implementations are byte-identical
    along a lockstep run, (2) reference blobs loaded into FRESH envs of both implementations (built
    with another seed) give the same frame and info immediately and the same trajectory afterwards,
    (3) which is also the trajectory the original envs continue on."""
    ref, dut = make_ref(0), make_dut(0)
    acts = mt19937_actions(0, num, 2 * steps)
    for t in range(steps):
        if t % check_every == 0:
            for e in range(num):
                assert ref.get_state(e) == dut.get_state(e), f"step {t} env {e}: state blobs differ"
        ref.act(acts[t])
        dut.act(acts[t])
        ref.observe()
        dut.observe()
    blobs = [ref.get_state(e) for e in range(num)]
    assert blobs == [dut.get_state(e) for e in range(num)]
    ref2, dut2 = make_ref(5), make_dut(5)
    for e in range(num):
        ref2.set_state(e, blobs[e])
        dut2.set_state(e, blobs[e])
    assert_same_observation(ref2, dut2, "after set_state")
    for t in range(steps, 2 * steps):
        ref.act(acts[t])
        ref2.act(acts[t])
        dut2.act(acts[t])
        assert_same_observation(ref2, dut2, t)
        r0, o0, f0 = ref.observe()
        r2, o2, f2 = ref2.observe()
        assert np.array_equal(o0["rgb"], o2["rgb"]) and np.array_equal(r0, r2) and np.array_equal(f0, f2)
    assert [ref2.get_state(e) for e in range(num)] == [dut2.get_state(e) for e in range(num)]
    for env in (ref, dut, ref2, dut2):
        env.close()


SNAP_SCRIPT = r"""
import sys
sys.path.insert(0, {root!r}); sys.path.insert(0, {root!r} + "/tests")
from helpers import make_pair, make_checked_pair, run_lockstep
pair = make_checked_pair if {checked!r} else make_pair
for name, mode in [("coinrun", "hard"), ("maze", "hard"), ("bigfish", "hard"), ("heist", "hard"), ("fruitbot", "hard")]:
    ref, dut = pair({lib!r}, 8, name, extra_options={{"snap_target_rect": False}}, distribution_mode=mode,
                         num_levels=200, start_level=0, rand_seed=0)
    run_lockstep(ref, dut, 200)
    ref.close(); dut.close()
print("SNAP_OFF_OK")
"""


def run_snap_off_lockstep(lib, checked=False):
    """The Qt-5-style un-snapped target rect (the known Qt 5 / Qt 6 risk, DESIGN §2) is a switch in both
    implementations; the oracle reads it from the environment once per process, hence the subprocess."""
    import subprocess
    import sys

    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ, QT_SHIM_SNAP="0")
    out = subprocess.run([sys.executable, "-c", SNAP_SCRIPT.format(root=root, lib=lib, checked=checked)], env=env, capture_output=True, text=True)
    assert "SNAP_OFF_OK" in out.stdout, out.stdout[-2000:] + out.stderr[-4000:]


# ---- pins of the raster restatement against a real Qt 6.6.3 raster engine. tests/golden/make_qt6_golden.py ran
# every case below through both and stored, in tests/golden/qt6/, 64-bit digests of Qt 6's results plus the few
# pixels where Qt 6 differs from the restatement; test_oracle.py replays the restatement against that record.
QT6_FRAME_CASES = {
    # case: ((game, mode) list, envs, steps, rand_seed, action seed, extra options)
    "raster": ([("coinrun", "hard"), ("bigfish", "hard"), ("maze", "hard"), ("jumper", "easy"), ("jumper", "hard"),
                ("fruitbot", "hard"), ("starpilot", "hard")], 8, 150, 3, 0, {}),
    "whole_world": ([("jumper", "easy"), ("jumper", "hard"), ("jumper", "memory"), ("coinrun", "hard"), ("caveflyer", "hard"),
                     ("climber", "hard"), ("ninja", "easy")], 4, 120, 5, 2, {"center_agent": False}),
    "rotated": ([("heist", "hard")], 8, 200, 3, 0, {}),
}


def digest64(arr):
    import hashlib

    return np.frombuffer(hashlib.sha256(np.ascontiguousarray(arr).tobytes()).digest()[:8], np.uint8)


def qt6_frame_runs(case, lib_path=None):
    """(game index, step, rgb batch) of every step of a QT6_FRAME_CASES case, from the oracle (or lib_path)."""
    games, n, steps, seed, aseed, extra = QT6_FRAME_CASES[case]
    for gi, (name, mode) in enumerate(games):
        env = RefVecEnv(n, name, distribution_mode=mode, num_levels=0, rand_seed=seed, lib_path=lib_path, **extra)
        acts = mt19937_actions(aseed, n, steps)
        for t in range(steps):
            env.act(acts[t])
            yield gi, t, env.observe()[1]["rgb"]
        env.close()


def _ellipse(lib, x, y, w, h, col, pw):
    import ctypes as C

    dst = np.full((64, 64), 0xff102030, np.uint32)
    lib.shim_test_draw_ellipse(dst.ctypes.data_as(C.c_void_p), 64, 64, C.c_double(x), C.c_double(y), C.c_double(w), C.c_double(h), *col, pw)
    return dst


def _line(lib, x1, y1, x2, y2, pw):
    import ctypes as C

    dst = np.full((64, 64), 0xff102030, np.uint32)
    lib.shim_test_draw_line(dst.ctypes.data_as(C.c_void_p), 64, 64, x1, y1, x2, y2, 252, 186, 3, pw)
    return dst


def ellipse_and_line_groups(lib):
    """drawEllipse (integer rects, pen / no pen / translucent brush, clipped by the device edge; jumper's compass
    discs on their non-integer rects) and drawLine(int...) with a cosmetic pen: (label, results) per group."""
    for x in range(-3, 60, 9):
        for y in range(-3, 60, 11):
            yield f"ellipses at ({x}, {y})", [_ellipse(lib, x, y, w, h, col, pw) for w in range(1, 20, 2) for h in (1, 2, 3, 8, 16, w)
                                             for col, pw in (((168, 166, 158, 255), 1), ((255, 255, 255, 120), -1), ((252, 186, 3, 255), 0))]
    # jumper's four compass discs (jumper.cpp:138-141): all but hard mode's centred one sit on non-integer rects
    unit = np.float32(64) / np.float32(12)
    easy = (float(np.float32(8.75) * unit), float(np.float32(.25) * unit), float(np.float32(3) * unit))
    world_easy = (53.60000228881836, 0.800000011920929, 9.600000381469727)   # center_agent=False, tests/tools/qt6_compass_mask.py
    world_hard = (60.400001525878906, 0.4000000059604645, 3.200000047683716)
    yield "compass discs", [_ellipse(lib, *rect, (168, 166, 158, 255), 1) for rect in
                            ((easy[0], easy[1], easy[2], easy[2]), (55.0, 1.0, 8.0, 8.0), world_easy + world_easy[2:], world_hard + world_hard[2:])]
    # every needle the compass can draw and more: all integer offsets within 9 px of in-bounds centres
    for cx, cy in ((54, 9), (59, 5), (20, 40), (10, 10)):
        yield f"lines from ({cx}, {cy})", [_line(lib, cx, cy, cx + dx, cy + dy, pw) for dx in range(-9, 10) for dy in range(-9, 10)
                                           if 0 <= cx + dx < 64 and 0 <= cy + dy < 64 for pw in (0, 1)]


def blit_and_fill_groups(lib, per_group=50):
    """Rules S and F on 1500 random rects, with positions and sizes deliberately placed on exact halves and
    quarters (qRound ties; Qt 6 rounds negative ties away from zero): (label, results) per `per_group` rects."""
    import ctypes as C

    rng = np.random.RandomState(7)
    srcs = [(np.arange(sw * sh, dtype=np.uint32).reshape(sh, sw)) | 0xff000000 for sw, sh in ((8, 8), (64, 64), (17, 17), (480, 270), (128, 64))]

    def draw(src, x, y, w, h):
        sh, sw = src.shape
        dst = np.zeros((64, 64), np.uint32)
        lib.shim_test_draw_image(dst.ctypes.data_as(C.c_void_p), 64, 64, src.ctypes.data_as(C.c_void_p), sw, sh, 0, C.c_double(x), C.c_double(y),
                                 C.c_double(w), C.c_double(h), C.c_double(0), C.c_double(1.0), 0)
        return dst

    def fill(x, y, w, h):
        dst = np.zeros((64, 64), np.uint32)
        lib.shim_test_fill_rect(dst.ctypes.data_as(C.c_void_p), 64, 64, C.c_double(x), C.c_double(y), C.c_double(w), C.c_double(h), 200, 100, 50)
        return dst

    def rnd():
        k = rng.randint(4)
        if k == 0:
            return float(rng.randint(-40, 100)) / 2
        if k == 1:
            return float(rng.randint(-80, 200)) / 4
        return rng.uniform(-20, 70)

    group = []
    for i in range(1500):
        x, y = rnd(), rnd()
        w = abs(rnd()) + 0.1 if rng.randint(2) else float(rng.randint(1, 80)) / 2
        h = abs(rnd()) + 0.1 if rng.randint(2) else float(rng.randint(1, 80)) / 2
        if rng.randint(3) == 0:
            w *= 4
            h *= 4
        src = srcs[rng.randint(len(srcs))]
        if not (w == src.shape[1] and h == src.shape[0]):  # 1:1 draws take Qt's unscaled path, which no in-scope draw call reaches
            group += [draw(src, x, y, w, h), fill(x, y, w, h)]
        if i % per_group == per_group - 1:
            yield f"rects {i + 1 - per_group}..{i}", group
            group = []
