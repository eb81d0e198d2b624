"""TEST INFRASTRUCTURE — ctypes driver for oracle/_ref/libenv_ref.so (the reference's own
game-logic sources compiled unmodified + the CPU raster restatement), speaking the libenv C ABI
exactly as gym3's CEnv would (vecgame.cpp:42-99, 437-457; option marshalling as env.py:110-124).

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference leg may
import this module.  Nothing here is on the product path.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REF_LIB = os.path.join(HERE, "_ref", "libenv_ref.so")
REF_LIB_QT6 = os.path.join(HERE, "_ref", "libenv_ref_qt6.so")

MAX_NAME = 128
MAX_NDIM = 16
DTYPE_UINT8, DTYPE_INT32, DTYPE_FLOAT32 = 1, 2, 3
SPACE_OBSERVATION, SPACE_ACTION, SPACE_INFO = 1, 2, 3
MAX_STATE_SIZE = 2 ** 20  # env.py:12


class _Value(C.Union):
    _fields_ = [("uint8", C.c_uint8), ("int32", C.c_int32), ("float32", C.c_float)]


class TensorType(C.Structure):
    _fields_ = [("name", C.c_char * MAX_NAME), ("scalar_type", C.c_int), ("dtype", C.c_int),
                ("shape", C.c_int * MAX_NDIM), ("ndim", C.c_int), ("low", _Value), ("high", _Value)]


class Option(C.Structure):
    _fields_ = [("name", C.c_char * MAX_NAME), ("dtype", C.c_int), ("count", C.c_int), ("data", C.c_void_p)]


class Options(C.Structure):
    _fields_ = [("items", C.POINTER(Option)), ("count", C.c_int)]


class Buffers(C.Structure):
    _fields_ = [("ob", C.POINTER(C.c_void_p)), ("rew", C.POINTER(C.c_float)), ("first", C.POINTER(C.c_uint8)),
                ("info", C.POINTER(C.c_void_p)), ("ac", C.POINTER(C.c_void_p))]


DISTRIBUTION_MODE = {"easy": 0, "hard": 1, "extreme": 2, "memory": 10}  # env.py:25-31, game.h:32-37


def default_pack():
    return os.path.join(os.path.dirname(HERE), "procgen_b200", "data", "assets.pack")


def make_options(keep, **kw):
    """kwargs -> libenv_options, like gym3's CEnv: str -> uint8[], bool -> uint8, int -> int32."""
    items = (Option * len(kw))()
    for i, (k, v) in enumerate(kw.items()):
        items[i].name = k.encode()
        if isinstance(v, str):
            buf = C.create_string_buffer(v.encode(), len(v.encode()))
            items[i].dtype, items[i].count = DTYPE_UINT8, len(v.encode())
        elif isinstance(v, bool):
            buf = (C.c_uint8 * 1)(int(v))
            items[i].dtype, items[i].count = DTYPE_UINT8, 1
        else:
            buf = (C.c_int32 * 1)(int(v))
            items[i].dtype, items[i].count = DTYPE_INT32, 1
        keep.append(buf)
        items[i].data = C.cast(buf, C.c_void_p)
    keep.append(items)
    return Options(items, len(kw))


class RefVecEnv:
    """The reference VecGame behind its libenv ABI. Defaults follow procgen/env.py:71-85,207-246."""

    def __init__(self, num, env_name, distribution_mode="hard", num_levels=0, start_level=0, rand_seed=0,
                 num_threads=0, center_agent=True, use_backgrounds=True, use_monochrome_assets=False,
                 restrict_themes=False, use_generated_assets=False, paint_vel_info=False,
                 use_sequential_levels=False, debug_mode=0, lib_path=None, pack_path=None, resource_root=None,
                 extra_options=None, launch_shape=None, ob_layout=None):
        """launch_shape=(chunks, serialize): a library that exports pgb200_set_launch_shape cuts every step,
        the initial reset included, into `chunks` env chunks per game (launches back to back if serialize).
        ob_layout: env e's observation goes to frame ob_layout[e] of a separate array (a non-contiguous
        set of observation pointers, as a caller with its own buffer layout passes them)."""
        lib_path = lib_path or REF_LIB
        if not os.path.exists(lib_path):
            raise FileNotFoundError(f"{lib_path} missing — run python oracle/build_ref.py in the build container")
        if os.path.basename(lib_path) == os.path.basename(REF_LIB_QT6):
            # real-Qt backend: satisfy Qt's unused DT_NEEDED entries with the empty stub libraries
            from oracle import qt6_support

            self.lib = C.CDLL(lib_path, handle=qt6_support.lazy_dlopen(lib_path))
        else:
            self.lib = C.CDLL(lib_path)
        L = self.lib
        L.libenv_make.restype = C.c_void_p
        L.libenv_make.argtypes = [C.c_int, Options]
        L.libenv_get_tensortypes.argtypes = [C.c_void_p, C.c_int, C.POINTER(TensorType)]
        L.libenv_set_buffers.argtypes = [C.c_void_p, C.POINTER(Buffers)]
        for f in (L.libenv_observe, L.libenv_act, L.libenv_close):
            f.argtypes = [C.c_void_p]
            f.restype = None
        if hasattr(L, "get_state"):
            L.get_state.argtypes = [C.c_void_p, C.c_int, C.c_char_p, C.c_int]
            L.get_state.restype = C.c_int
            L.set_state.argtypes = [C.c_void_p, C.c_int, C.c_char_p, C.c_int]
            L.set_state.restype = None
        self.num = num
        self._keep = []
        self._ob_layout = None
        opts = dict(
            env_name=env_name, num_levels=num_levels, start_level=start_level, num_actions=15,
            use_sequential_levels=bool(use_sequential_levels), debug_mode=debug_mode, rand_seed=rand_seed,
            num_threads=num_threads, render_human=False,
            resource_root=resource_root if resource_root is not None else (pack_path or default_pack()) + ":",
            center_agent=bool(center_agent), use_generated_assets=bool(use_generated_assets),
            use_monochrome_assets=bool(use_monochrome_assets), restrict_themes=bool(restrict_themes),
            use_backgrounds=bool(use_backgrounds), paint_vel_info=bool(paint_vel_info),
            distribution_mode=DISTRIBUTION_MODE[distribution_mode])
        opts.update(extra_options or {})
        self.h = L.libenv_make(num, make_options(self._keep, **opts))
        if launch_shape is not None and hasattr(L, "pgb200_set_launch_shape"):
            L.pgb200_set_launch_shape.argtypes = [C.c_void_p, C.c_int, C.c_int]
            L.pgb200_set_launch_shape.restype = None
            L.pgb200_set_launch_shape(self.h, int(launch_shape[0]), int(bool(launch_shape[1])))
        n_info = L.libenv_get_tensortypes(self.h, SPACE_INFO, None)
        info_types = (TensorType * n_info)()
        L.libenv_get_tensortypes(self.h, SPACE_INFO, info_types)
        self.info_names = [t.name.decode() for t in info_types]
        self.rgb = np.zeros((num, 64, 64, 3), np.uint8)
        self.rew = np.zeros(num, np.float32)
        self.first = np.zeros(num, np.uint8)
        self.ac = np.zeros(num, np.int32)
        self.info = {}
        info_ptrs = (C.c_void_p * (n_info * num))()
        for si, t in enumerate(info_types):
            dt = {DTYPE_UINT8: np.uint8, DTYPE_INT32: np.int32, DTYPE_FLOAT32: np.float32}[t.dtype]
            arr = np.zeros(num, dt)
            self.info[t.name.decode()] = arr
            for e in range(num):
                info_ptrs[si * num + e] = arr.ctypes.data + e * arr.itemsize
        if ob_layout is None:
            ob_ptrs = (C.c_void_p * num)(*[self.rgb.ctypes.data + e * 64 * 64 * 3 for e in range(num)])
        else:
            # the caller's observation slots are not one contiguous [num][64][64][3] block: env e writes
            # frame ob_layout[e] of a larger array, and self.rgb is the env-ordered view of it
            self._ob_store = np.zeros((int(max(ob_layout)) + 1, 64, 64, 3), np.uint8)
            ob_ptrs = (C.c_void_p * num)(*[self._ob_store.ctypes.data + int(s) * 64 * 64 * 3 for s in ob_layout])
            self._ob_layout = np.asarray(ob_layout)
        ac_ptrs = (C.c_void_p * num)(*[self.ac.ctypes.data + e * 4 for e in range(num)])
        self._bufs = Buffers(ob_ptrs, self.rew.ctypes.data_as(C.POINTER(C.c_float)),
                             self.first.ctypes.data_as(C.POINTER(C.c_uint8)), info_ptrs, ac_ptrs)
        self._keep += [ob_ptrs, ac_ptrs, info_ptrs]
        L.libenv_set_buffers(self.h, C.byref(self._bufs))

    def observe(self):
        self.lib.libenv_observe(self.h)
        if self._ob_layout is not None:
            self.rgb[:] = self._ob_store[self._ob_layout]
        return self.rew, {"rgb": self.rgb}, self.first

    def act(self, ac):
        self.ac[:] = np.asarray(ac, dtype=np.int32)
        self.lib.libenv_act(self.h)

    def get_info(self):
        return [{k: v[i] for k, v in self.info.items()} for i in range(self.num)]

    def get_state(self, idx):
        buf = C.create_string_buffer(MAX_STATE_SIZE)
        n = self.lib.get_state(self.h, idx, buf, MAX_STATE_SIZE)
        return buf.raw[:n]

    def set_state(self, idx, blob):
        self.lib.set_state(self.h, idx, blob, len(blob))

    def close(self):
        if self.h:
            self.lib.libenv_close(self.h)
            self.h = None


def mt19937_actions(seed, num, steps, n_actions=15):
    """Action recipe of SURVEY §8c: ac[t][i] = g() % 15 drawn env-major per step from mt19937(seed)."""
    rs = np.random.RandomState(seed)  # MT19937 with init_genrand(seed) == std::mt19937(seed)
    raw = rs.randint(0, 2 ** 32, size=(steps, num), dtype=np.uint32).astype(np.uint64)
    return (raw % n_actions).astype(np.int32)
