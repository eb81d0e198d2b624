"""ProcgenGym3Env on the GPU — host-side mirror of the reference's Python boundary.

Mirrors ``procgen/env.py``: ``BaseProcgenEnv`` (:66-200) + ``ProcgenGym3Env`` (:203-246) with the same
constructor keywords, defaults, option marshalling and the gym3 ``Env`` surface callers use
(``num``, ``ob_space``, ``ac_space``, ``observe()``, ``act()``, ``get_info()``, ``callmethod()``).
Differences, all on purpose:

* ``observe()`` returns ``torch.cuda`` tensors that alias the library's HBM buffers (no copy, no
  host round trip); ``act()`` accepts a CUDA tensor (stays on device) or anything array-like.
* ``host_buffers=True`` selects the reference's exact contract instead: numpy buffers owned by
  the caller, filled through ``libenv_set_buffers/act/observe`` like gym3's ``CEnv`` does.
* ``shard=(rank, world_size)`` makes this handle own envs ``[rank*num, (rank+1)*num)`` of one
  logical ``world_size*num``-env VecGame (same per-env seed chain, vecgame.cpp:301-314);
  ``gather_observations()`` is the single NCCL gather of SURVEY §8(e).

gym3 is not installable here, so the few space types used are defined below with gym3's names.
"""
from __future__ import annotations

import ctypes as C
import os
import random
from dataclasses import dataclass
from typing import List, Optional, Sequence, Tuple

import numpy as np

from . import libenv as L

MAX_STATE_SIZE = 2 ** 20  # env.py:12

ENV_NAMES = [  # env.py:14-31
    "bigfish", "bossfight", "caveflyer", "chaser", "climber", "coinrun", "dodgeball", "fruitbot",
    "heist", "jumper", "leaper", "maze", "miner", "ninja", "plunder", "starpilot",
]

EXPLORATION_LEVEL_SEEDS = {  # env.py:33-42
    "coinrun": 1949448038, "caveflyer": 1259048185, "leaper": 1318677581, "jumper": 1434825276,
    "maze": 158988835, "heist": 876640971, "climber": 1561126160, "ninja": 1123500215,
}

DISTRIBUTION_MODE_DICT = {"easy": 0, "hard": 1, "extreme": 2, "memory": 10, "exploration": 20}  # env.py:45-51


# ---- the slice of gym3.types the reference's callers touch
@dataclass(frozen=True)
class Discrete:
    n: int
    dtype_name: str = "int32"


@dataclass(frozen=True)
class TensorType:
    eltype: Discrete
    shape: Tuple[int, ...]


class DictType(dict):
    pass


def create_random_seed():
    """env.py:54-63 (mpi4py de-correlation becomes torch.distributed rank de-correlation)."""
    rand_seed = random.SystemRandom().randint(0, 2 ** 31 - 1)
    try:
        import torch.distributed as dist

        if dist.is_available() and dist.is_initialized():
            rand_seed = rand_seed - (rand_seed % dist.get_world_size()) + dist.get_rank()
    except Exception:
        pass
    return rand_seed


def _broadcast_seed(seed):
    try:
        import torch
        import torch.distributed as dist

        if dist.is_available() and dist.is_initialized():
            dev = "cuda" if dist.get_backend() == "nccl" else "cpu"
            t = torch.tensor([seed], dtype=torch.int64, device=dev)
            dist.broadcast(t, src=0)
            return int(t.item())
    except Exception:
        pass
    raise ValueError("shard=(rank, world) needs an explicit rand_seed when torch.distributed is not initialised")


class _CudaArray:
    """Minimal __cuda_array_interface__ holder so torch can alias library-owned HBM."""

    def __init__(self, ptr, shape, typestr):
        self.__cuda_array_interface__ = {"shape": tuple(shape), "typestr": typestr, "data": (int(ptr), False),
                                         "version": 2, "strides": None}


class BaseProcgenEnv:
    """env.py:66-200."""

    def __init__(self, num, env_name, options, debug=False, rand_seed=None, num_levels=0, start_level=0,
                 use_sequential_levels=False, debug_mode=0, resource_root=None, num_threads=4, render_mode=None,
                 host_buffers=False, device=None, shard=None, snap_target_rect=True, lib_path=None):
        self._lib = L.load(lib_path)
        self.combos = self.get_combos()
        if render_mode is None:
            render_human = False
        elif render_mode == "rgb_array":
            render_human = True
        else:
            raise Exception(f"invalid render mode {render_mode}")
        if render_human:
            raise NotImplementedError("render_mode='rgb_array' (512x512 antialiased info['rgb']) is out of scope")
        if rand_seed is None:
            rand_seed = create_random_seed()
            if shard is not None:
                # every shard of one logical VecGame must replay the SAME per-env seed chain
                # (vecgame.cpp:301-314): take rank 0's draw instead of de-correlating per rank
                rand_seed = _broadcast_seed(rand_seed)
        if resource_root is None:
            resource_root = os.path.join(os.path.dirname(os.path.abspath(__file__)), "data") + os.sep

        options = dict(options)
        options.update({
            "env_name": env_name,
            "num_levels": num_levels,
            "start_level": start_level,
            "num_actions": len(self.combos),
            "use_sequential_levels": bool(use_sequential_levels),
            "debug_mode": debug_mode,
            "rand_seed": rand_seed,
            "num_threads": num_threads,
            "render_human": render_human,
            "resource_root": resource_root,
        })
        self._host_buffers = bool(host_buffers)
        self._torch = None
        self._next_level_seeds = None
        self._final_outputs = None
        self._pause_mask = None
        self._action_repeat = None
        self._rollout = None
        self._snapshots = None
        self._num_levels, self._start_level = num_levels, start_level
        self._consumer_slot = None
        self._graph_stepped = False   # act() has run inside a CUDA graph capture
        self._retired_consumers = []  # consumer buffers a captured graph may still write
        self._timing = False
        if self._lib.pgb200_is_device_build():
            import torch

            self._torch = torch
            if not torch.cuda.is_available():
                raise RuntimeError("procgen_b200 needs a CUDA device (there is no CPU fallback)")
            if device is None:
                device = torch.cuda.current_device()
            device = torch.device(device).index if not isinstance(device, int) else device
            options["cuda_device"] = int(device)
        self.device_index = device
        if shard is not None:
            rank, world = shard
            options["env_index_offset"] = int(rank) * int(num)
            options["env_index_total"] = int(world) * int(num)
        self.shard = shard
        if not snap_target_rect:
            options["snap_target_rect"] = False
        self.options = options
        self.num = int(num)

        self._keep = []
        self._h = self._lib.libenv_make(self.num, L.make_options(self._keep, options))
        if not self._h:
            raise RuntimeError("libenv_make failed")

        # spaces (vecgame.cpp:212-268); the action space is unwrapped like env.py:138
        self.ob_space = DictType(rgb=TensorType(Discrete(256, "uint8"), (64, 64, 3)))
        self.ac_space = TensorType(Discrete(len(self.combos), "int32"), ())
        self._info_names = ["prev_level_seed", "prev_level_complete", "level_seed"]

        if self._host_buffers:
            self._setup_host_buffers()
        else:
            self._setup_device_buffers()

    # ------------------------------------------------------------------ buffer plumbing
    def _setup_host_buffers(self):
        n = self.num
        self._rgb = None
        if self._torch is not None:
            try:
                # page-locked from the start (cudaHostAlloc through torch): the library then DMAs straight
                # into it without having to register 12 KiB/env of pageable memory
                self._rgb_pinned = self._torch.zeros((n, 64, 64, 3), dtype=self._torch.uint8, pin_memory=True)
                self._rgb = self._rgb_pinned.numpy()
            except Exception:
                self._rgb = None
        if self._rgb is None:
            self._rgb = np.zeros((n, 64, 64, 3), np.uint8)
        self._rew = np.zeros(n, np.float32)
        self._first = np.zeros(n, np.uint8)
        self._ac = np.zeros(n, np.int32)
        self._info = {"prev_level_seed": np.zeros(n, np.int32), "prev_level_complete": np.zeros(n, np.uint8),
                      "level_seed": np.zeros(n, np.int32)}
        ob_ptrs = (C.c_void_p * n)(*[self._rgb.ctypes.data + e * 64 * 64 * 3 for e in range(n)])
        ac_ptrs = (C.c_void_p * n)(*[self._ac.ctypes.data + e * 4 for e in range(n)])
        info_ptrs = (C.c_void_p * (3 * n))()
        for si, name in enumerate(self._info_names):
            arr = self._info[name]
            for e in range(n):
                info_ptrs[si * n + e] = arr.ctypes.data + e * arr.itemsize
        self._bufs = L.Buffers(ob_ptrs, self._rew.ctypes.data_as(C.POINTER(C.c_float)),
                               self._first.ctypes.data_as(C.POINTER(C.c_uint8)), info_ptrs, ac_ptrs)
        self._keep += [ob_ptrs, ac_ptrs, info_ptrs]
        self._lib.libenv_set_buffers(self._h, C.byref(self._bufs))

    def _alias(self, ptr, shape, typestr):
        """CUDA tensor aliasing library-owned device memory at `ptr` (an address or a ctypes pointer)."""
        if not isinstance(ptr, int):
            ptr = C.cast(ptr, C.c_void_p).value
        return self._torch.as_tensor(_CudaArray(ptr, shape, typestr), device=self._torch.device("cuda", self.device_index))

    def _setup_device_buffers(self):
        torch = self._torch
        if torch is None:
            raise RuntimeError("device-resident buffers need the CUDA build")
        dev = torch.device("cuda", self.device_index)
        with torch.cuda.device(dev):
            self._stream_handle = torch.cuda.current_stream(dev).cuda_stream
            self._lib.pgb200_set_stream(self._h, C.c_void_p(self._stream_handle))
            db = L.DeviceBuffers()
            rc = self._lib.pgb200_get_device_buffers(self._h, C.byref(db))
            if rc != 0:
                raise RuntimeError("pgb200_get_device_buffers failed")
            n = self.num
            self._rgb = self._alias(db.rgb, (n, 64, 64, 3), "|u1")
            self._rew = self._alias(db.rew, (n,), "<f4")
            self._first = self._alias(db.first, (n,), "|u1")
            self._ac = self._alias(db.action, (n,), "<i4")
            self._info = {"prev_level_seed": self._alias(db.prev_level_seed, (n,), "<i4"),
                          "prev_level_complete": self._alias(db.prev_level_complete, (n,), "|u1"),
                          "level_seed": self._alias(db.level_seed, (n,), "<i4")}
        self._dev = dev
        self._pinned_ac = None

    # ------------------------------------------------------------------ gym3 Env surface
    def observe(self):
        """-> (rew f32[N], {"rgb": u8[N,64,64,3]}, first bool[N]); device tensors unless host_buffers."""
        if self._host_buffers:
            self._refuse_in_capture("observe")
            self._lib.libenv_observe(self._h)
            return self._rew, {"rgb": self._rgb}, self._first.astype(bool)
        return self._rew, {"rgb": self._rgb}, self._first.bool()

    # ------------------------------------------------------------------ CUDA graph capture
    def _capturing(self) -> bool:
        return self._torch is not None and self._torch.cuda.is_current_stream_capturing()

    def _refuse_in_capture(self, method: str) -> None:
        if self._capturing():
            raise RuntimeError(f"procgen_b200: {method}() cannot run inside CUDA graph capture (it waits for the GPU or "
                               "allocates); call it before the capture or after it")

    def _wait_for_replays(self) -> None:
        """Before a call that reads or writes env state from the host: once this handle has been captured, its
        steps may also be graph replays on the caller's current stream, which the handle's own stream does not
        see. Rebinding to that stream waits for both."""
        if self._graph_stepped and not self._host_buffers:
            with self._torch.cuda.device(self._dev):
                cur = self._torch.cuda.current_stream(self._dev).cuda_stream
                self._lib.pgb200_set_stream(self._h, C.c_void_p(cur))
                self._stream_handle = cur
                self._lib.pgb200_sync(self._h)

    def act(self, ac):
        """env.py:197-200: actions are cast to int32. Asynchronous, like VecGame::act.

        Inside ``torch.cuda.graph`` (or any capture on the current stream) act() takes a CUDA tensor only and
        the step becomes part of the graph: the handle is rebound to the capture stream without a host wait,
        and every replay steps the envs again with whatever the action tensor then holds. Set up before the
        capture what the step should use (next_level_seeds(), pause_mask(), action_repeat(), enable_consumer_output(),
        rollout(), set_launch_shape()): a graph keeps the launch shape, the level choice, the pause mask, the action
        repeat, the consumer output and the rollout it was captured with."""
        if self._capturing():
            if self._host_buffers:
                raise RuntimeError("procgen_b200: act() cannot be captured in a CUDA graph with host_buffers=True; "
                                   "use the device-resident handle")
            if not (self._torch.is_tensor(ac) and ac.is_cuda):
                raise RuntimeError("procgen_b200: act() inside CUDA graph capture takes a CUDA tensor of actions; "
                                   "host arrays need a synchronised copy that cannot be captured")
            if getattr(self, "_peer", None) is not None:
                raise RuntimeError("procgen_b200: act() cannot be captured while enable_peer_gather() is on: the mirror "
                                   "buffer alternates on the host")
            if self._timing:
                raise RuntimeError("procgen_b200: act() cannot be captured between kernel_timing_begin() and kernel_timing_end()")
            self._graph_stepped = True
        if self._host_buffers:
            self._ac[:] = np.asarray(ac).astype(np.int32)
            for arr in (self._next_level_seeds, self._pause_mask, self._action_repeat):
                if arr is not None:
                    # libenv_act reads the level choices, the pause mask and the repeat counts on the library's
                    # own stream: the caller's torch writes must be complete first
                    self._torch.cuda.current_stream(arr.device).synchronize()
                    break
            self._lib.libenv_act(self._h)
            return
        torch = self._torch
        with torch.cuda.device(self._dev):
            # keep every launch on the caller's current stream (a capture stream included: the library rebinds
            # to a capturing stream without waiting)
            cur = torch.cuda.current_stream(self._dev).cuda_stream
            if cur != self._stream_handle:
                self._lib.pgb200_set_stream(self._h, C.c_void_p(cur))
                self._stream_handle = cur
            if torch.is_tensor(ac) and ac.is_cuda:
                self._ac.copy_(ac.to(torch.int32), non_blocking=True)
            else:
                host = torch.as_tensor(np.asarray(ac).astype(np.int32))
                if self._pinned_ac is None:
                    # two pinned staging buffers, each guarded by an event recorded behind its H2D copy:
                    # act() never rewrites host memory a still-queued DMA is going to read
                    self._pinned_ac = [torch.empty(self.num, dtype=torch.int32, pin_memory=True) for _ in range(2)]
                    self._pinned_ev = [torch.cuda.Event(), torch.cuda.Event()]
                    self._pinned_used = [False, False]
                    self._pinned_i = 0
                i = self._pinned_i
                self._pinned_i = 1 - i
                if self._pinned_used[i]:
                    self._pinned_ev[i].synchronize()
                self._pinned_ac[i].copy_(host)
                self._ac.copy_(self._pinned_ac[i], non_blocking=True)
                self._pinned_ev[i].record(torch.cuda.current_stream(self._dev))
                self._pinned_used[i] = True
            self._lib.pgb200_act_device(self._h)

    def get_info(self) -> List[dict]:
        """gym3's list-of-dicts form (env.py:128-136). One D2H copy for all three columns; callers on
        the hot path should use get_info_tensors() (columns, no copy) instead."""
        self._refuse_in_capture("get_info")
        if self._host_buffers:
            cols = [self._info[k].tolist() for k in self._info_names]
        else:
            torch = self._torch
            packed = torch.stack([self._info[k].to(torch.int32) for k in self._info_names]).cpu().numpy()
            cols = [packed[0].tolist(), packed[1].astype(np.uint8).tolist(), packed[2].tolist()]
        a, b, c3 = self._info_names
        return [{a: x, b: y, c3: z} for x, y, z in zip(*cols)]

    def get_info_tensors(self):
        """Column form of get_info() without a host copy."""
        return dict(self._info)

    def next_level_seeds(self):
        """int32 CUDA tensor [num] aliasing the library's per-env choice of the next level (allocated, all -1,
        on the first call). At every reset inside a step (episode end, timeout, or action -1) env e checks its
        entry s: s >= 0 starts the new level with seed s — any seed in [0, 2**31), also outside
        [start_level, start_level + num_levels) — and the step sets the entry back to -1 (an override is used
        once); s = -1 leaves the reset as it is (a draw from the env's own level seed generator, which an
        override does not advance, or the +997 of use_sequential_levels). The initial reset is not affected:
        to start envs on chosen levels, write seeds and act() with action -1 for them. get_state / set_state
        neither read nor change the array.

        Write it with torch ops on the stream you step on (device-resident mode); with host_buffers=True,
        act() waits for the current torch stream before it starts the step.

        A CUDA graph reads the array only if it was requested before the capture: call this once first. Inside
        the capture the tensor may then be refilled with torch ops like any other input of the graph."""
        if self._next_level_seeds is None:
            self._refuse_in_capture("next_level_seeds")
            torch = self._torch
            ptr = C.POINTER(C.c_int32)()
            with torch.cuda.device(self.device_index):
                if self._lib.pgb200_get_next_level_seeds(self._h, C.byref(ptr)) != 0:
                    raise RuntimeError("pgb200_get_next_level_seeds failed")
                self._next_level_seeds = self._alias(ptr, (self.num,), "<i4")
        return self._next_level_seeds

    def final_outputs(self):
        """{"rgb": uint8 [num, 64, 64, 3], "level_end": uint8 [num]}: CUDA tensors aliasing the library's final
        outputs (allocated, zero-filled, on the first call; from then on every step fills them). A step that ends
        an episode resets the env inside it and returns the next level's first frame; after every step,
        level_end[e] says whether env e's level ended in it and why: 0 it did not, 1 (LEVEL_END_GAME) the game
        ended it (death or completion; prev_level_complete tells which), 2 (LEVEL_END_TIMEOUT) the step limit,
        a truncation whose final state a learner bootstraps from, 3 (LEVEL_END_CALLER) action -1. Where
        level_end[e] != 0, rgb[e] is the frame of the state the level ended in; elsewhere it keeps its value.
        level_end != 0 exactly where first is set, except that under use_sequential_levels a completed level
        continues with first = 0 and reports 1. Everything else the step outputs is unchanged.

        A CUDA graph fills them only if they were requested before the capture: call this once first."""
        if self._final_outputs is None:
            self._refuse_in_capture("final_outputs")
            torch = self._torch
            out = L.FinalOutputs()
            with torch.cuda.device(self.device_index):
                if self._lib.pgb200_get_final_outputs(self._h, C.byref(out)) != 0:
                    raise RuntimeError("pgb200_get_final_outputs failed")
                self._final_outputs = {"rgb": self._alias(out.rgb, (self.num, 64, 64, 3), "|u1"),
                                       "level_end": self._alias(out.level_end, (self.num,), "|u1")}
        return dict(self._final_outputs)

    def pause_mask(self):
        """uint8 CUDA tensor [num] aliasing the library's per-env pause mask (allocated, all 0, on the first call). In
        every step, env e with mask[e] != 0 is paused: its state stays as it is, byte for byte (a paused step does
        not count toward the time limit), its action (-1 included) is ignored and its next_level_seeds() entry is
        neither read nor consumed; its rgb and info slots keep their values, and rew[e] = 0, first[e] = 0 (and
        final_outputs()["level_end"][e] = 0). With the consumer output on, the stack of a paused env repeats the
        frame it is paused on. Every other env steps exactly as it would without the mask. A step does not clear
        the mask: an entry stays in force until the caller clears it. get_state / set_state neither read nor
        change it.

        Write it with torch ops on the stream you step on (device-resident mode); with host_buffers=True, act()
        waits for the current torch stream before it starts the step.

        A CUDA graph reads the mask only if it was requested before the capture: call this once first. Inside the
        capture the tensor may then be refilled with torch ops like any other input of the graph."""
        if self._pause_mask is None:
            self._refuse_in_capture("pause_mask")
            torch = self._torch
            ptr = C.POINTER(C.c_uint8)()
            with torch.cuda.device(self.device_index):
                if self._lib.pgb200_get_pause_mask(self._h, C.byref(ptr)) != 0:
                    raise RuntimeError("pgb200_get_pause_mask failed")
                self._pause_mask = self._alias(ptr, (self.num,), "|u1")
        return self._pause_mask

    def action_repeat(self):
        """int32 CUDA tensor [num] aliasing the library's per-env action repeat counts (allocated, all 1, on the first
        call). In every step, env e with entry r plays max(r, 1) game steps with its action and stops after the first
        whose level ends (game end, time limit, action -1, or a completed level with use_sequential_levels), so
        action -1 plays one. rew[e] is the float32 sum of those game steps' rewards, in order; first[e], the info
        slots and final_outputs()["level_end"][e] are the last one's, and rgb[e] is the frame of the final state
        (final_outputs()["rgb"][e] that of the state the level ended in). The env takes its next_level_seeds() entry
        at the one reset a step can contain. A paused env (pause_mask()) plays no game step. The rollout and the
        consumer output move on once per act(). A step does not change the array; get_state / set_state, snapshots,
        the level bank and lookahead neither read nor change it. An all-ones array steps exactly as a handle that
        never called this.

        Write it with torch ops on the stream you step on (device-resident mode); with host_buffers=True, act()
        waits for the current torch stream before it starts the step.

        A CUDA graph reads the array only if it was requested before the capture: call this once first. Inside the
        capture the tensor may then be refilled with torch ops like any other input of the graph."""
        if self._action_repeat is None:
            self._refuse_in_capture("action_repeat")
            torch = self._torch
            ptr = C.POINTER(C.c_int32)()
            with torch.cuda.device(self.device_index):
                if self._lib.pgb200_get_action_repeat(self._h, C.byref(ptr)) != 0:
                    raise RuntimeError("pgb200_get_action_repeat failed")
                self._action_repeat = self._alias(ptr, (self.num,), "<i4")
        return self._action_repeat

    def rollout(self, slots: int):
        """{"rgb": uint8 [slots, num, 64, 64, 3], "rew": float32 [slots, num], "first": uint8 [slots, num], "cursor": int32
        [1]}: CUDA tensors aliasing the library's rollout, a ring of `slots` copies of the step outputs. From the first
        call on, every step (eager or replayed from a CUDA graph) moves cursor c on to (c + 1) % slots on the device and
        stores its rgb, rew and first into slot c from the render kernel itself, byte for byte what observe() returns,
        so a learner's rollout storage needs no copy after the step. The first call writes the current outputs into
        slot 0 and sets cursor to 0. With final_outputs() a slot holds the next level's first frame (what rgb holds);
        a paused env's slot holds the frame it is paused on, with rew = 0 and first = 0. get_state / set_state leave
        the rollout alone. A rollout of T steps plus the observation to bootstrap from needs slots >= T + 1.

        The memory (12 KiB per env and slot) is held until close(); there is no off switch, and `slots` is fixed by
        the first call (ValueError for another value, or for slots < 2). A CUDA graph fills the rollout only if it
        was requested before the capture: call this once first."""
        slots = int(slots)
        if self._rollout is not None:
            if slots != self._rollout["rgb"].shape[0]:
                raise ValueError(f"rollout(): this handle's rollout has {self._rollout['rgb'].shape[0]} slots")
            return dict(self._rollout)
        if slots < 2:
            raise ValueError("rollout(): slots must be at least 2")
        self._refuse_in_capture("rollout")
        self._wait_for_replays()
        torch = self._torch
        out = L.Rollout()
        with torch.cuda.device(self.device_index):
            if self._lib.pgb200_get_rollout(self._h, slots, C.byref(out)) != 0:
                raise RuntimeError("pgb200_get_rollout failed")
            n = self.num
            self._rollout = {"rgb": self._alias(out.rgb, (slots, n, 64, 64, 3), "|u1"),
                             "rew": self._alias(out.rew, (slots, n), "<f4"),
                             "first": self._alias(out.first, (slots, n), "|u1"),
                             "cursor": self._alias(out.cursor, (1,), "<i4")}
        return dict(self._rollout)

    def snapshots(self, slots: int):
        """{"save_from": int32 [slots], "load_from": int32 [num], "source": int32 [slots]}: CUDA tensors aliasing the
        library's snapshot slots, a store of `slots` env states kept on the device (allocated, every entry -1, on the
        first call). Write env indices into save_from and slot indices into load_from with torch ops on the stream you
        step on, then call apply_snapshots(): slot s takes the state of env save_from[s], then env e takes the state of
        slot load_from[e] and is observed as set_state observes it. Each applied entry reads -1 afterwards; an entry
        that cannot be applied (out of range, an empty slot, a slot holding another game's state) keeps its value, so
        `(load_from >= 0).any()` finds them. source[s] is the env whose state slot s holds, -1 while it is empty. A
        loaded env is a byte-for-byte copy of the source env at save time: get_state() returns the blob the source
        had, and it steps on as the source would have.

        Each slot is sized for the largest live state of the handle's games (about 80 KB for coinrun), held until
        close(); `slots` is fixed by the first call (ValueError for another value, or for slots < 1). The first call
        cannot run inside a CUDA graph capture; the tensors may then be refilled inside one. Slots are not portable
        across handles or processes: get_state() is the portable form."""
        slots = int(slots)
        if self._snapshots is not None:
            if slots != self._snapshots["save_from"].shape[0]:
                raise ValueError(f"snapshots(): this handle's store has {self._snapshots['save_from'].shape[0]} slots")
            return dict(self._snapshots)
        if slots < 1:
            raise ValueError("snapshots(): slots must be at least 1")
        self._refuse_in_capture("snapshots")
        self._wait_for_replays()
        torch = self._torch
        out = L.Snapshots()
        with torch.cuda.device(self.device_index):
            if self._lib.pgb200_get_snapshots(self._h, slots, C.byref(out)) != 0:
                raise RuntimeError(f"pgb200_get_snapshots failed: {slots} slots could not be allocated")
            self._snapshots = {"save_from": self._alias(out.save_from, (slots,), "<i4"),
                               "load_from": self._alias(out.load_from, (self.num,), "<i4"),
                               "source": self._alias(out.source, (slots,), "<i4")}
        return dict(self._snapshots)

    def apply_snapshots(self) -> None:
        """Apply the saves and loads written into snapshots()' arrays: every save first, then every load, then the
        loaded envs' observations, on the current torch stream (as act(), it rebinds the handle to it). It never waits
        for the host, so it may run inside torch.cuda.graph; a replay applies the arrays as they are then. Envs not
        loaded, the rollout, final outputs, the pause mask, next_level_seeds(), the bank and lookahead are untouched."""
        if self._snapshots is None:
            raise RuntimeError("apply_snapshots(): call snapshots(slots) first")
        torch = self._torch
        if self._host_buffers:
            self._refuse_in_capture("apply_snapshots")
            # the library works on its own stream here: the caller's torch writes must be complete first, and its
            # reads of the arrays must see the apply
            torch.cuda.current_stream(self._snapshots["save_from"].device).synchronize()
            rc = self._lib.pgb200_apply_snapshots(self._h)
            self._lib.pgb200_sync(self._h)
        else:
            with torch.cuda.device(self._dev):
                cur = torch.cuda.current_stream(self._dev).cuda_stream
                if cur != self._stream_handle:
                    self._lib.pgb200_set_stream(self._h, C.c_void_p(cur))
                    self._stream_handle = cur
                if self._capturing():
                    self._graph_stepped = True
                rc = self._lib.pgb200_apply_snapshots(self._h)
        if rc != 0:
            raise RuntimeError("pgb200_apply_snapshots failed")

    def build_level_bank(self, seeds=None, capacity: int = 0) -> None:
        """Bank the levels of `seeds` (default: range(start_level, start_level + num_levels)) for every game of the
        handle: a reset inside a step onto a banked seed copies the level generated here instead of generating it
        again. Only speed changes: every output and state is the one a handle without a bank gives. The first call
        fixes the capacity at max(len(seeds), capacity) distinct seeds, which must not be 0; a later call rebuilds
        the bank in place (CUDA graphs captured after the first call see the rebuild), and an empty `seeds` empties
        it. The rebuild is ordered behind every step issued before it, graph replays on the current stream
        included. Raises ValueError for a seed outside [0, 2^31), more distinct seeds than the capacity, or a first
        call with no seeds and no capacity."""
        if seeds is None:
            if self._num_levels == 0:
                raise ValueError("build_level_bank(): num_levels == 0 plays unboundedly many levels; pass the seeds to bank")
            seeds = range(self._start_level, self._start_level + self._num_levels)
        self._refuse_in_capture("build_level_bank")
        self._wait_for_replays()
        arr = np.asarray(list(seeds), dtype=np.int64).reshape(-1)
        if arr.size and (arr.min() < 0 or arr.max() >= 2 ** 31):
            raise ValueError("build_level_bank(): every seed must be in [0, 2^31)")
        arr = np.ascontiguousarray(arr.astype(np.int32))
        ptr = arr.ctypes.data_as(C.POINTER(C.c_int32))
        if self._lib.pgb200_build_level_bank(self._h, ptr, int(arr.size), int(capacity)) != 0:
            raise ValueError(f"build_level_bank(): {len(np.unique(arr))} distinct seeds exceed the bank's capacity, or a "
                             "first call has no seeds and capacity 0")

    def level_bank_info(self) -> dict:
        """{"levels": distinct seeds banked, "bytes": device memory the bank holds}; zeros without a bank."""
        self._refuse_in_capture("level_bank_info")
        levels, nbytes = C.c_int(0), C.c_int64(0)
        self._lib.pgb200_level_bank_info(self._h, C.byref(levels), C.byref(nbytes))
        return {"levels": levels.value, "bytes": nbytes.value}

    def enable_level_lookahead(self) -> None:
        """Generate each env's next level while its current episode plays (level lookahead), for num_levels = 0 and
        any other level set a bank does not hold: an env's next seed is known when its episode starts, so its level is
        generated into a slot of its own beside the frames of a step, and the reset at the episode's end copies it
        instead of generating it inside the step. Only speed changes: every output and state is the one a handle
        without lookahead gives. A prediction can miss (next_level_seeds() overrides, set_state, a completed level of
        use_sequential_levels): that reset generates as before. A bank, where there is one, serves its seeds first.

        Memory: one slot per env, sized by its game (24-77 KB; about 5 GB for coinrun at 65 536 envs), and staging,
        held until close(); level_lookahead_info()["bytes"] reports it. There is no off switch. The call generates every
        env's next level before it returns; a second call does nothing. CUDA graphs captured after it use lookahead,
        ones captured before it never do."""
        self._refuse_in_capture("enable_level_lookahead")
        self._wait_for_replays()
        if self._lib.pgb200_enable_level_lookahead(self._h) != 0:
            raise RuntimeError("pgb200_enable_level_lookahead failed")

    def level_lookahead_info(self) -> dict:
        """{"served": resets served from a lookahead slot, "bank": resets served from the bank, "generated": resets
        that generated their level (the three counted from enable_level_lookahead() on), "bytes": device memory
        lookahead holds}; zeros without lookahead."""
        self._refuse_in_capture("level_lookahead_info")
        self._wait_for_replays()
        out = (C.c_int64 * 4)()
        if self._lib.pgb200_level_lookahead_info(self._h, out) != 0:
            raise RuntimeError("pgb200_level_lookahead_info failed")
        return dict(zip(("served", "bank", "generated", "bytes"), list(out)))

    def callmethod(self, method: str, *args, **kwargs):
        return getattr(self, method)(*args, **kwargs)

    def _state_envs(self, envs, method):
        """envs (default: every env, in order) as a contiguous int32 array; ValueError for an index out of range"""
        if envs is None:
            return np.arange(self.num, dtype=np.int32)
        arr = np.asarray(envs, dtype=np.int64).reshape(-1)
        if arr.size and (arr.min() < 0 or arr.max() >= self.num):
            raise ValueError(f"{method}(): env indices must be in [0, {self.num})")
        return np.ascontiguousarray(arr.astype(np.int32))

    def get_state(self, envs=None):
        """One bytes blob per listed env (default: every env, in order) in the reference's wire format (env.py:139-147,
        vecgame.cpp:437-445). An env may be listed more than once. One library call gathers every listed env's state on
        the device and writes the blobs on the host."""
        self._refuse_in_capture("get_state")
        self._wait_for_replays()
        arr = self._state_envs(envs, "get_state")
        data, offsets = C.c_void_p(), C.POINTER(C.c_int64)()
        if self._lib.pgb200_get_states(self._h, arr.ctypes.data_as(C.POINTER(C.c_int32)), int(arr.size), C.byref(data),
                                       C.byref(offsets)) != 0:
            raise RuntimeError("pgb200_get_states failed")
        if arr.size == 0:
            return []
        offs = np.ctypeslib.as_array(offsets, shape=(arr.size + 1,)).tolist()
        return [C.string_at(data.value + offs[i], offs[i + 1] - offs[i]) for i in range(arr.size)]

    def set_state(self, states, envs=None):
        """Load states[i] into env envs[i] (default: every env, in order; env.py:149-153, vecgame.cpp:447-457). Each
        listed env's observation, rew, first and info are refreshed from its restored state; the other envs are
        untouched. ValueError for an env out of range or listed twice, or a number of blobs other than of envs. One
        library call restores every listed env; a malformed blob ends the process with `fatal: set_state:`."""
        self._refuse_in_capture("set_state")
        self._wait_for_replays()
        arr = self._state_envs(envs, "set_state")
        states = [bytes(st) for st in states]
        if len(states) != arr.size:
            raise ValueError(f"set_state(): {len(states)} states for {arr.size} envs")
        if np.unique(arr).size != arr.size:
            raise ValueError("set_state(): an env is listed twice")
        offsets = np.zeros(arr.size + 1, np.int64)
        np.cumsum([len(st) for st in states], out=offsets[1:])
        if self._lib.pgb200_set_states(self._h, arr.ctypes.data_as(C.POINTER(C.c_int32)), int(arr.size), b"".join(states),
                                       offsets.ctypes.data_as(C.POINTER(C.c_int64))) != 0:
            raise RuntimeError("pgb200_set_states failed")

    def get_combos(self):  # env.py:155-172
        return [("LEFT", "DOWN"), ("LEFT",), ("LEFT", "UP"), ("DOWN",), (), ("UP",), ("RIGHT", "DOWN"), ("RIGHT",),
                ("RIGHT", "UP"), ("D",), ("A",), ("W",), ("S",), ("Q",), ("E",)]

    def keys_to_act(self, keys_list: Sequence[Sequence[str]]) -> List[Optional[np.ndarray]]:  # env.py:174-195
        result = []
        for keys in keys_list:
            action = None
            max_len = -1
            for i, combo in enumerate(self.get_combos()):
                pressed = all(key in keys for key in combo)
                if pressed and (max_len < len(combo)):
                    action = i
                    max_len = len(combo)
            if action is not None:
                action = np.array([action])
            result.append(action)
        return result

    # ------------------------------------------------------------------ GPU extras
    def sync(self):
        self._refuse_in_capture("sync")
        self._lib.pgb200_sync(self._h)

    def errors(self) -> int:
        """OR of the per-env sticky error bits (0 = healthy)."""
        self._refuse_in_capture("errors")
        self._wait_for_replays()
        return int(self._lib.pgb200_get_errors(self._h, None))

    def kernel_launches(self) -> int:
        """Kernel launches issued so far; a step captured in a CUDA graph counts once, not per replay."""
        return int(self._lib.pgb200_kernel_launches(self._h))

    def set_launch_shape(self, chunks: int = 0, serialize: bool = False) -> None:
        """Measurement knob (see pgb200_set_launch_shape): env chunks per step, launches back to back."""
        self._refuse_in_capture("set_launch_shape")
        self._lib.pgb200_set_launch_shape(self._h, int(chunks), int(bool(serialize)))

    def kernel_timing_begin(self, max_launch_pairs: int) -> None:
        """Bracket every (logic, render) kernel pair with CUDA events until kernel_timing_end()."""
        self._refuse_in_capture("kernel_timing_begin")
        if self._lib.pgb200_kernel_timing_begin(self._h, int(max_launch_pairs)) != 0:
            raise RuntimeError("procgen_b200: kernel timing is not available on a handle with final_outputs()")
        self._timing = True

    def kernel_timing_end(self) -> dict:
        import ctypes as C

        self._refuse_in_capture("kernel_timing_end")
        out = (C.c_double * 5)()
        pairs = int(self._lib.pgb200_kernel_timing_end(self._h, out))
        self._timing = False
        return {"logic_ms": out[0], "render_ms": out[1], "setup_ms": out[4], "launch_pairs": pairs, "env_steps": out[3]}

    def enable_peer_gather(self, dst: int = 0) -> bool:
        """Turn gather_observations() into peer writes: allocate the gathered array as torch symmetric
        memory (every rank maps every rank's copy over NVLink), hand the library the address of this
        shard's slot in `dst`'s copy, and let every render launch be followed by a copy of its frames
        to that slot (pgb200_set_rgb_mirror) — the transfer then overlaps the rest of the step and
        gather_observations() only has to run one cross-rank barrier. Collective (call on all ranks).
        Returns False (and keeps the NCCL gather) when symmetric memory cannot be set up."""
        import torch.distributed as dist

        self._refuse_in_capture("enable_peer_gather")
        torch = self._torch
        world, rank = dist.get_world_size(), dist.get_rank()
        ok = torch.zeros(1, device=self._dev, dtype=torch.int32)
        try:
            import torch.distributed._symmetric_memory as symm_mem

            n = self.num
            frame = 64 * 64 * 3
            buf = symm_mem.empty((2 * world * n * frame,), dtype=torch.uint8, device=self._dev)
            hdl = symm_mem.rendezvous(buf, dist.group.WORLD)
            ptr = int(hdl.buffer_ptrs[dst])
            slots = [ptr + (b * world * n + rank * n) * frame for b in (0, 1)]
            self._peer = {"buf": buf, "hdl": hdl, "dst": dst, "slots": slots,
                          "views": [buf[b * world * n * frame:(b + 1) * world * n * frame].view(world * n, 64, 64, 3) for b in (0, 1)]}
            ok += 1
        except Exception as e:  # noqa: BLE001 - any failure means: keep the collective
            self._peer_error = repr(e)
        dist.all_reduce(ok, op=dist.ReduceOp.MIN)
        if int(ok.item()) != 1:
            self._peer = None
            return False
        with torch.cuda.device(self._dev):
            self._lib.pgb200_set_rgb_mirror(self._h, C.c_void_p(self._peer["slots"][0]), C.c_void_p(self._peer["slots"][1]))
        return True

    def gather_observations(self, dst: int = 0):
        """The only cross-rank exchange on this path (SURVEY §8e): every rank's rgb shard on `dst`.
        Returns u8[world*num,64,64,3] on dst, None elsewhere. After enable_peer_gather() the frames
        were already written into dst's memory behind each render launch and this is one barrier;
        otherwise it is one NCCL gather."""
        import torch.distributed as dist

        torch = self._torch
        world = dist.get_world_size()
        peer = getattr(self, "_peer", None)
        if peer is not None and peer["dst"] == dst:
            peer["hdl"].barrier(channel=0)   # on the current stream: every rank's copies of this step have landed
            if dist.get_rank() == dst:
                return peer["views"][int(self._lib.pgb200_mirror_parity(self._h))]
            return None
        if dist.get_rank() == dst:
            out = getattr(self, "_gather_buf", None)
            if out is None or out.shape[0] != world * self.num:
                out = self._gather_buf = torch.empty((world * self.num, 64, 64, 3), dtype=torch.uint8, device=self._dev)
            dist.gather(self._rgb, list(out.chunk(world, dim=0)), dst=dst)
            return out
        dist.gather(self._rgb, None, dst=dst)
        return None

    # ------------------------------------------------------------------ consumer epilogue (SURVEY §8(f)4)
    def enable_consumer_output(self, dtype=None, frames: int = 1):
        """Have the render kernel also write what a learner feeds its network: rgb / 255 as float16 or
        bfloat16, planar CHW, `frames` frames stacked along the channel axis with baselines'
        VecFrameStack reset rule (an env that starts an episode sees zeros for the older frames).
        consumer_observation() then returns [num, 3*frames, 64, 64] without any further kernel.

        A CUDA graph keeps the buffer, dtype and frames it was captured with: enable the output before the
        capture, and capture again after changing it."""
        self._refuse_in_capture("enable_consumer_output")
        torch = self._torch
        dtype = dtype or torch.float16
        code = {torch.float16: 1, torch.bfloat16: 2}[dtype]
        slots = 1 if frames == 1 else 2 * frames
        if self._graph_stepped and getattr(self, "_consumer", None) is not None:
            # a graph captured earlier still writes the old buffer: never hand its memory to anything else
            self._retired_consumers.append(self._consumer)
        with torch.cuda.device(self._dev):
            self._consumer = torch.zeros((self.num, slots, 3, 64, 64), dtype=dtype, device=self._dev)
            self._consumer_k = int(frames)
            torch.cuda.current_stream(self._dev).synchronize()
            rc = self._lib.pgb200_set_consumer_output(self._h, C.c_void_p(self._consumer.data_ptr()), code, int(frames))
        if rc != 0:
            raise ValueError("pgb200_set_consumer_output rejected the arguments")

    def consumer_observation(self):
        """[num, 3*frames, 64, 64] view (oldest frame first) of the consumer output; valid until the next act().

        Once the handle has been stepped inside a CUDA graph, graph replays move the ring on the device only,
        so from then on (and inside the capture) this is a copy gathered through consumer_slot_tensor(),
        without a host wait, instead of a view."""
        k = self._consumer_k
        if k == 1:
            return self._consumer[:, 0]
        if self._graph_stepped or self._capturing():
            torch = self._torch
            idx = self.consumer_slot_tensor().to(torch.int64) + 1 + torch.arange(k, device=self._dev)
            return self._consumer.index_select(1, idx).reshape(self.num, 3 * k, 64, 64)
        s = int(self._lib.pgb200_consumer_slot(self._h))
        return self._consumer[:, s + 1:s + 1 + k].reshape(self.num, 3 * k, 64, 64)

    def consumer_slot_tensor(self):
        """int32 CUDA tensor [1] aliasing the device-resident ring position s of the consumer output: the slot the
        latest step wrote, advanced on the device by every step, eager or replayed from a CUDA graph. The ordered
        stack (oldest frame first) is ring slots s + 1 .. s + k of the [num, 2k, 3, 64, 64] ring (k > 1), so a
        captured policy reads it without the host:

            slot, ring = env.consumer_slot_tensor(), env.consumer_ring()   # before the capture
            ar = torch.arange(k, device="cuda")
            with torch.cuda.graph(g):
                env.act(actions)
                idx = slot.long() + 1 + ar
                obs = ring.index_select(1, idx).reshape(env.num, 3 * k, 64, 64)
                logits = policy(obs)

        (consumer_observation() does the same once the handle has been captured.) Written on the stream the
        handle steps on."""
        if self._consumer_slot is None:
            ptr = C.POINTER(C.c_int32)()
            if self._lib.pgb200_get_consumer_slot_device(self._h, C.byref(ptr)) != 0:
                raise RuntimeError("pgb200_get_consumer_slot_device failed")
            self._consumer_slot = self._alias(ptr, (1,), "<i4")
        return self._consumer_slot

    def consumer_ring(self):
        """The consumer output's ring itself: [num, slots, 3, 64, 64] (slots = 1 for frames == 1, else 2 * frames)."""
        return self._consumer

    def gather_how(self) -> str:
        if getattr(self, "_peer", None) is not None:
            return ("peer writes: each render launch is followed by a copy of its frames into rank-0 symmetric memory over "
                    "NVLink (pgb200_set_rgb_mirror); gather = one symmetric-memory barrier per step")
        return "torch.distributed.gather (NCCL) of the rgb shard after the step" + (
            f" (peer path unavailable: {self._peer_error})" if getattr(self, "_peer_error", None) else "")

    def close(self):
        if getattr(self, "_consumer", None) is not None and getattr(self, "_h", None):
            self._lib.pgb200_set_consumer_output(self._h, None, 0, 0)
            self._consumer = None
        if getattr(self, "_peer", None) is not None and getattr(self, "_h", None):
            self._lib.pgb200_set_rgb_mirror(self._h, None, None)
            self._peer = None
        if getattr(self, "_h", None):
            self._next_level_seeds = None
            self._final_outputs = None
            self._pause_mask = None
            self._action_repeat = None
            self._rollout = None
            self._snapshots = None
            self._lib.libenv_close(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class ProcgenGym3Env(BaseProcgenEnv):
    """env.py:203-246 — same keywords and defaults."""

    def __init__(self, num, env_name, center_agent=True, use_backgrounds=True, use_monochrome_assets=False,
                 restrict_themes=False, use_generated_assets=False, paint_vel_info=False, distribution_mode="hard",
                 **kwargs):
        assert distribution_mode in DISTRIBUTION_MODE_DICT, f'"{distribution_mode}" is not a valid distribution mode.'
        if distribution_mode == "exploration":
            assert env_name in EXPLORATION_LEVEL_SEEDS, f"{env_name} does not support exploration mode"
            distribution_mode = DISTRIBUTION_MODE_DICT["hard"]
            assert "num_levels" not in kwargs, "exploration mode overrides num_levels"
            kwargs["num_levels"] = 1
            assert "start_level" not in kwargs, "exploration mode overrides start_level"
            kwargs["start_level"] = EXPLORATION_LEVEL_SEEDS[env_name]
        else:
            distribution_mode = DISTRIBUTION_MODE_DICT[distribution_mode]
        options = {
            "center_agent": bool(center_agent),
            "use_generated_assets": bool(use_generated_assets),
            "use_monochrome_assets": bool(use_monochrome_assets),
            "restrict_themes": bool(restrict_themes),
            "use_backgrounds": bool(use_backgrounds),
            "paint_vel_info": bool(paint_vel_info),
            "distribution_mode": distribution_mode,
        }
        super().__init__(num, env_name, options, **kwargs)
