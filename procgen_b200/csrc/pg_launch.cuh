// Kernels, launch wrappers and the per-game dispatch table. Included by pg_runtime.cu (host runtime +
// C ABI) and by one translation unit per game (games_tu/tu_<game>.cu), so the 16 games compile in
// parallel; a game's kernels are instantiated only in its own unit.
#pragma once
#include <stdarg.h>
#include <stddef.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <type_traits>

#include "pg_kernels.cuh"

#ifndef PG_HOSTSIM
#include <cuda_runtime.h>
#endif

namespace pg {

// ================================================================= errors (cpp-utils.cpp:8-20)
static inline void pg_fatal(const char *fmt, ...) {
    fprintf(stderr, "fatal: ");
    va_list args;
    va_start(args, fmt);
    vfprintf(stderr, fmt, args);
    va_end(args);
    exit(EXIT_FAILURE);
}
#define pg_fassert(cond)                                                                  \
    do {                                                                                  \
        if (!(cond)) {                                                                    \
            fprintf(stderr, "fassert failed '%s' at %s:%d\n", #cond, __FILE__, __LINE__); \
            exit(EXIT_FAILURE);                                                           \
        }                                                                                 \
    } while (0)

#ifndef PG_HOSTSIM
#define CUDA_CHECK(expr)                                                                          \
    do {                                                                                          \
        cudaError_t _e = (expr);                                                                  \
        if (_e != cudaSuccess)                                                                    \
            pg_fatal("CUDA error %s at %s:%d: %s\n", cudaGetErrorName(_e), __FILE__, __LINE__, cudaGetErrorString(_e)); \
    } while (0)
using Stream = cudaStream_t;
using Event = cudaEvent_t;
#else
// the host debug build has no streams or events: members of these types stay null there
struct HostStream;
struct HostEvent;
using Stream = HostStream *;
using Event = HostEvent *;
#endif

// ================================================================= kernels
// Two launches per step:
//   logic_kernel   one WARP per env. All 32 lanes execute the serial game logic redundantly and in
//                  lockstep (every load/store is warp-uniform), and fan out only inside
//                  pg_scan_down, which turns the reference's O(E) entity-collision loops into E/32
//                  ballots. A warp, not a thread, is the unit so unrelated envs never diverge
//                  against each other and dozens of envs per SM hide each other's load latency.
//   render_kernel  one CTA per env: blit-list build + per-pixel gather + packed RGB store
#ifndef PG_LOGIC_WARPS
#define PG_LOGIC_WARPS 2
#endif
#ifndef PG_LOGIC_MIN_BLOCKS
#define PG_LOGIC_MIN_BLOCKS 24
#endif
#ifndef PG_STEP_CHUNKS
#define PG_STEP_CHUNKS 8
#endif
#ifndef PG_AUX_STREAMS
#define PG_AUX_STREAMS 16   // one per game of the 16-game list: the slow games (level generation) must not queue behind each other
#endif
constexpr int kLogicThreads = 32 * PG_LOGIC_WARPS;  // one warp = one env; few warps per CTA so a finished
constexpr int kLogicEnvsPerBlock = PG_LOGIC_WARPS;  // env frees its slot without waiting on many siblings
constexpr int kRenderThreads = 128;

#ifndef PG_HOSTSIM
// Persistent: the grid is sized to fill the machine once and every warp pulls env indices from a
// global ticket counter until the launch's range is exhausted, so a long env (level reset) only
// delays its own warp and no SM slot idles waiting for a block launch.
// FINAL: phase A of a step with final outputs; an env whose level ends is appended to p.reset_list.
// PAUSE: the handle has a pause mask. A paused env's warp reads its entry, writes its outputs and takes the next
// ticket without touching the env's state; it never enters phase B's list.
// REPEAT: the handle has action repeat. A warp plays up to repeat[env] game steps of its env; the tickets spread the
// uneven work as they spread level generation.
template <class G, bool INIT, bool LEVEL_CHOICE = false, bool FINAL = false, bool PAUSE = false, bool REPEAT = false>
__global__ void __launch_bounds__(kLogicThreads, PG_LOGIC_MIN_BLOCKS) logic_kernel(KParams p, unsigned int *ticket) {
    using Frame = typename FrameFor<G>::type;
    const unsigned lane = threadIdx.x & 31u;
    while (true) {
        unsigned t = 0;
        if (lane == 0)
            t = atomicAdd(ticket, 1u);
        t = __shfl_sync(0xffffffffu, t, 0);
        if (t >= (unsigned)p.env_count)
            break;
        const int env = p.env_first + (int)t * p.env_step;
        const long long t0 = p.dbg_cycles ? clock64() : 0;
        env_logic<G, Frame, INIT, LEVEL_CHOICE, FINAL, PAUSE, REPEAT>(p, env);
        __syncwarp();
        if (p.dbg_cycles && lane == 0)
            p.dbg_cycles[env] = (uint32_t)(clock64() - t0);
    }
}

// Phase B of a step with final outputs: the resets of the envs phase A listed. Persistent and ticketed like the
// logic kernel, because level generation runs here (milliseconds for caveflyer, jumper and leaper).
// BANK: the handle has a level bank; the only kernel a banked step adds to those of an unbanked one.
// LOOK: the handle has level lookahead: resets copy from the env's lookahead slot where it holds their level, and list
// the envs whose next level lookahead_kernel generates.
// REPEAT: the handle has action repeat; a reset's reward joins the sum phase A left in rew.
template <class G, bool BANK = false, bool LOOK = false, bool REPEAT = false>
__global__ void __launch_bounds__(kLogicThreads, PG_LOGIC_MIN_BLOCKS) finish_kernel(KParams p, unsigned int *ticket) {
    using Frame = typename FrameFor<G>::type;
    const unsigned lane = threadIdx.x & 31u;
    const unsigned count = *p.reset_count;
    while (true) {
        unsigned t = 0;
        if (lane == 0)
            t = atomicAdd(ticket, 1u);
        t = __shfl_sync(0xffffffffu, t, 0);
        if (t >= count)
            break;
        const int env = p.reset_list[t];
        // a banked step's reset runs here: its cycles join phase A's in the profiling aid
        const long long t0 = ((BANK || LOOK) && p.dbg_cycles) ? clock64() : 0;
        env_finish_logic<G, Frame, BANK, LOOK, REPEAT>(p, env);
        __syncwarp();
        if ((BANK || LOOK) && p.dbg_cycles && lane == 0)
            p.dbg_cycles[env] += (uint32_t)(clock64() - t0);
    }
}

// Level bank build: warp w generates the levels w, w + warps, ... of p.bank into their slots, in the staging area
// stage + w * bank_stage_bytes(p) (the bank's memory budget bounds how many warps run)
template <class G>
__global__ void __launch_bounds__(kLogicThreads) bank_build_kernel(KParams p, unsigned char *stage, int count, int warps) {
    const int w = (int)((blockIdx.x * blockDim.x + threadIdx.x) >> 5);
    if (w >= warps)
        return;
    for (int item = w; item < count; item += warps) {
        bank_generate_level<G>(p, p.bank, p.bank.seeds[item], [&] { return p.bank.slots + (size_t)item * p.bank.slot_bytes; },
                               stage + (size_t)w * bank_stage_bytes(p));
        __syncwarp();
    }
}

// Level lookahead: the levels of the envs p.look.list holds (count[0] of them), generated into their slots. Persistent
// with a fixed grid of p.look.stage_warps warps, each with its own staging area, ticketed over the list by count[1];
// the count is read on the device, so a step that launches it stays capturable.
template <class G>
__global__ void __launch_bounds__(kLogicThreads) lookahead_kernel(KParams p, unsigned int *count) {
    const int w = (int)((blockIdx.x * blockDim.x + threadIdx.x) >> 5);
    if (w >= p.look.stage_warps)
        return;
    const unsigned lane = threadIdx.x & 31u;
    const unsigned n = count[0];
    unsigned char *stage = p.look.stage + (size_t)w * bank_stage_bytes(p);
    while (true) {
        unsigned t = 0;
        if (lane == 0)
            t = atomicAdd(count + 1, 1u);
        t = __shfl_sync(0xffffffffu, t, 0);
        if (t >= n)
            break;
        lookahead_generate<G>(p, (int)t, stage);
        __syncwarp();
    }
}

// Level lookahead's bulk fill: one warp per env of the launch predicts its next level (lookahead_predict)
template <class G>
__global__ void __launch_bounds__(kLogicThreads) lookahead_predict_kernel(KParams p) {
    const int i = (int)((blockIdx.x * blockDim.x + threadIdx.x) >> 5);
    if (i < p.env_count)
        lookahead_predict(p, p.env_first + i * p.env_step, p.bank.slots != nullptr);
}

// Frame setup: one warp per env (4 envs per block). Everything about a frame that is O(entities +
// cell columns): camera, visible window, per-column / per-row pixel spans, background, overlay and
// entity blits (incl. the scan conversion of rotated sprites). Every warp of the grid runs this
// same code, which is what the instruction cache wants; the render kernel that follows — one CTA
// per env — is left with the O(pixels + cells) work and picks the result up with one bulk copy.
// Each warp builds its env's FrameSetupT in its own slot of the block's shared memory — the record's
// counters are shared-memory atomics and its read-backs shared-memory loads — and stores the FrameSharedT
// prefix to the env's global record once, at the end.
constexpr int kSetupThreads = 128;
#ifndef PG_SETUP_MIN_BLOCKS
#define PG_SETUP_MIN_BLOCKS 8   // 64 registers x 32 warps/SM: more envs in flight beat more registers (96 x 20 was slower)
#endif
// Resident setup blocks per SM: PG_SETUP_MIN_BLOCKS, or as many as the warps' records (shared memory) allow;
// the register cap follows (65536 / (128 * blocks)).
template <class G, int VIEW>
struct SetupTune {
    static constexpr int kSmemBytes = (int)sizeof(typename FrameFor<G, VIEW>::setup) * (kSetupThreads / 32);
    // 227 KiB usable per SM, 1 KiB reserved per resident CTA, 128 B of static shared memory (build_entity_blits)
    static constexpr int kFit = (227 * 1024) / (kSmemBytes + 1024 + 128);
    static constexpr int kMinBlocks = kFit >= PG_SETUP_MIN_BLOCKS ? PG_SETUP_MIN_BLOCKS : (kFit >= 1 ? kFit : 1);
};
// LIST: phase B of a step with final outputs, the warps of the grid stride over p.reset_list (which never holds a
// paused env). PAUSE: a paused env's warp returns; its frame_setup slot goes stale, and nothing reads it.
template <class G, int VIEW, bool LIST = false, bool PAUSE = false>
__global__ void __launch_bounds__(kSetupThreads, SetupTune<G, VIEW>::kMinBlocks) setup_kernel(KParams p) {
    using Setup = typename FrameFor<G, VIEW>::setup;
    extern __shared__ __align__(128) unsigned char smem_raw[];
    Setup &f = reinterpret_cast<Setup *>(smem_raw)[threadIdx.x >> 5];
    const int lane = (int)(threadIdx.x & 31u);
    const int i = (int)blockIdx.x * (kSetupThreads / 32) + (int)(threadIdx.x >> 5);
    if (LIST) {
        const int count = (int)*p.reset_count;
        for (int j = i; j < count; j += (int)gridDim.x * (kSetupThreads / 32)) {
            const int env = p.reset_list[j];
            env_setup_frame<G, Setup>(p, env, f, lane, 32);
            __syncwarp();
            PG_SETUP_PHASE_BEGIN;
            env_store_frame<Setup>(p, env, f);  // ends with a __syncwarp: the next env may reuse the slot
            PG_SETUP_PHASE(9);
        }
        return;
    }
    if (i >= p.env_count)
        return;
    const int env = p.env_first + i * p.env_step;
    if (PAUSE && p.paused[env])
        return;
    env_setup_frame<G, Setup>(p, env, f, lane, 32);
    __syncwarp();
    PG_SETUP_PHASE_BEGIN;
    env_store_frame<Setup>(p, env, f);
    PG_SETUP_PHASE(9);
}

#ifndef PG_RENDER_CTAS_PER_SM
#define PG_RENDER_CTAS_PER_SM 0  // 0 = as many as registers / the frame allow
#endif
// Resident CTAs per SM the render kernel is compiled for: as many as the frame (shared memory)
// allows; the register cap follows (65536 / (128 * CTAs)).
template <class G, int VIEW>
struct RenderTune {
    static constexpr size_t kFrameBytes = sizeof(typename FrameFor<G, VIEW>::type);
#ifdef PG_RENDER_MIN_BLOCKS
    static constexpr int kMinBlocks = PG_RENDER_MIN_BLOCKS;
#else
    // 227 KiB usable per SM, 1 KiB reserved per resident CTA
    static constexpr int kFit = (int)((227 * 1024) / (kFrameBytes + 1024 + 16));
    // the games that draw grid cells run best at 7 CTAs (72 registers: at 64 the gather loop spills),
    // the entity-only games at 8
    static constexpr int kWant = G::DRAWS_GRID ? 7 : 8;
    static constexpr int kMinBlocks = kFit >= kWant ? kWant : (kFit >= 1 ? kFit : 1);
#endif
};

// ---- async-proxy plumbing (PTX): mbarrier + bulk copies (the TMA engine's 1-D mode; SASS UBLKCP)
__device__ __forceinline__ uint32_t pg_smem_addr(const void *ptr) { return (uint32_t)__cvta_generic_to_shared(ptr); }
__device__ __forceinline__ void pg_mbar_init(unsigned long long *bar, unsigned count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(pg_smem_addr(bar)), "r"(count) : "memory");
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void pg_mbar_arrive_expect_tx(unsigned long long *bar, unsigned bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(pg_smem_addr(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void pg_mbar_wait(unsigned long long *bar, unsigned parity) {
    unsigned done = 0;
    while (!done) {  // try_wait suspends the thread in hardware for a while before it returns false
        asm volatile(
            "{\n"
            ".reg .pred p;\n"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
            "selp.u32 %0, 1, 0, p;\n"
            "}\n"
            : "=r"(done)
            : "r"(pg_smem_addr(bar)), "r"(parity)
            : "memory");
    }
}
// global -> shared, completion counted on the mbarrier; 16-byte aligned, size a multiple of 16
__device__ __forceinline__ void pg_bulk_load(void *dst_smem, const void *src_gmem, unsigned bytes, unsigned long long *bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(pg_smem_addr(dst_smem)),
                 "l"(src_gmem), "r"(bytes), "r"(pg_smem_addr(bar))
                 : "memory");
}
// shared -> global, queued in the thread's current bulk group
__device__ __forceinline__ void pg_bulk_store(void *dst_gmem, const void *src_smem, unsigned bytes) {
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(dst_gmem), "r"(pg_smem_addr(src_smem)), "r"(bytes) : "memory");
}
// returns once the engine has read the sources of the stores queued so far (the CTA may then exit / reuse them)
__device__ __forceinline__ void pg_bulk_commit_and_wait() {
    asm volatile("cp.async.bulk.commit_group;" ::: "memory");
    asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
}

// One CTA renders one env's frame:
//   stage                  warp 0 arms the mbarrier and queues the bulk copies: what the setup kernel prepared
//                          (spans, background, counts, cell map, lookups) and one per pre-scaled tile (global
//                          table -> shared arena)
//   compose                warp w owns rows y = w (mod 4): gather (cells over background; a lane = 4 pixel
//                          columns x 8 rows), then paint the entity blits in draw order, lanes sharing each blit
//   pack + store           RGB32 -> RGB888 in place, one bulk copy of the 12 KiB frame to the observation buffer
//                          (and, with a rollout, a second one to the env's rollout slot, in the same bulk group)
// render_env_frame is that sequence for the env env_of() returns, on mbarrier phase `parity`. PASS: see
// render_kernel. The env index and whether phase A's env ended its level are fetched where they are needed, so
// that nothing stays live across the frame (the 8-CTA games have no register to spare). ROLL: see render_kernel.
template <class G, int VIEW, int PASS, bool ROLL, class EnvOf>
__device__ __forceinline__ void render_env_frame(const KParams &p, typename FrameFor<G, VIEW>::type &f, EnvOf env_of, unsigned parity) {
    using Frame = typename FrameFor<G, VIEW>::type;
    const int tid = (int)threadIdx.x;
#ifdef PG_PHASE_TIMING
    long long t0 = clock64(), t1;
#define PG_RENDER_PHASE(id)                                       \
    do {                                                          \
        t1 = clock64();                                           \
        if (tid == 0)                                             \
            p.hdr[env_of()].dbg_phase[id] = (uint32_t)(t1 - t0);       \
        t0 = t1;                                                  \
    } while (0)
#else
#define PG_RENDER_PHASE(id) do { } while (0)
#endif
    using Shared = typename FrameFor<G, VIEW>::shared;
    const Shared *gs = reinterpret_cast<const Shared *>(p.frame_setup + (size_t)env_of() * p.frame_setup_stride);
    if (tid < 32) {
        // Everything the setup kernel prepared for this env — one bulk copy into the head of the frame —
        // and the pre-scaled tiles its cells need, one bulk copy each, all counted on one mbarrier phase.
        const int nj = G::DRAWS_GRID ? (gs->n_tjobs < MAX_TILE_JOBS ? gs->n_tjobs : MAX_TILE_JOBS) : 0;
        unsigned words = 0;
        for (int j = tid; j < nj; j += 32) words += gs->tjob_words[j];
        for (int d = 16; d > 0; d >>= 1) words += __shfl_xor_sync(0xffffffffu, words, d);
        if (tid == 0) {
            pg_mbar_arrive_expect_tx(&f.mbar, (unsigned)sizeof(Shared) + 4u * words);
            pg_bulk_load(static_cast<Shared *>(&f), gs, (unsigned)sizeof(Shared), &f.mbar);
        }
        __syncwarp();
        for (int j = tid; j < nj; j += 32)
            pg_bulk_load(f.arena + gs->tjob_dst[j], p.tiles.texels + gs->tjob_src[j], 4u * gs->tjob_words[j], &f.mbar);
    }
    pg_mbar_wait(&f.mbar, parity);
    PG_RENDER_PHASE(0);
    // warp w owns rows y = w (mod warps): gather and paint need no block barrier in between
    env_render_compose<G, Frame>(p, f, tid >> 5, kRenderThreads >> 5, tid & 31, 32);
    __syncthreads();
    PG_RENDER_PHASE(5);
    if (p.consumer != nullptr && !is_final_frame<PASS>(p, env_of())) {
        // Consumer epilogue: the frame as normalised 16-bit floats, planar, into ring slot s (and its
        // twin s + k); an env that starts an episode this step gets the older frames of its window
        // zeroed (the frame-stack convention of baselines' VecFrameStack). Thread = pixel pairs.
        const int kf = p.consumer_k, s = *p.consumer_slot_dev;
        const int slots = kf == 1 ? 1 : 2 * kf;
        uint32_t *base = reinterpret_cast<uint32_t *>(p.consumer) + (size_t)env_of() * slots * (3 * RES_W * RES_H / 2);
        const uint16_t *lut = p.consumer_lut;
        for (int pair = tid; pair < RES_W * RES_H / 2; pair += kRenderThreads) {
            const uint32_t c0 = f.fb[2 * pair], c1 = f.fb[2 * pair + 1];
#pragma unroll
            for (int ch = 0; ch < 3; ch++) {
                const int sh = 16 - 8 * ch;  // R, G, B planes
                const uint32_t v = (uint32_t)lut[(c0 >> sh) & 0xffu] | ((uint32_t)lut[(c1 >> sh) & 0xffu] << 16);
                base[(size_t)(s * 3 + ch) * (RES_W * RES_H / 2) + pair] = v;
                if (kf > 1)
                    base[(size_t)((s + kf) * 3 + ch) * (RES_W * RES_H / 2) + pair] = v;
            }
        }
        if (kf > 1 && p.first[env_of()]) {
            // window of this step = ring slots s+1 .. s+k (the newest is s+k); zero the k-1 older ones
            // wherever they live: slot j and its twin j +- k
            for (int j = 1; j < kf; j++) {
                const int a = (s + j) % kf;
                for (int w = tid; w < 3 * RES_W * RES_H / 2; w += kRenderThreads) {
                    base[(size_t)a * (3 * RES_W * RES_H / 2) + w] = 0u;
                    base[(size_t)(a + kf) * (3 * RES_W * RES_H / 2) + w] = 0u;
                }
            }
        }
    }
    {
        // RGB32 -> RGB888 in place: every thread reads its 8 pixel quads, then (barrier) writes them packed
        constexpr int kQuadsPerThread = RES_W * RES_H / 4 / kRenderThreads;
        uint32_t c[kQuadsPerThread][4];
#pragma unroll
        for (int j = 0; j < kQuadsPerThread; j++) {
            const uint4 v = reinterpret_cast<const uint4 *>(f.fb)[tid + j * kRenderThreads];
            c[j][0] = v.x; c[j][1] = v.y; c[j][2] = v.z; c[j][3] = v.w;
        }
        __syncthreads();
#pragma unroll
        for (int j = 0; j < kQuadsPerThread; j++) Raster<G, Frame>::pack_quad(c[j], f.fb + 3 * (tid + j * kRenderThreads));
    }
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // generic-proxy writes of f.fb -> visible to the bulk copy
    __syncthreads();
    PG_RENDER_PHASE(6);
    if (tid == 0) {
        pg_bulk_store((is_final_frame<PASS>(p, env_of()) ? p.final_rgb : p.rgb) + (size_t)env_of() * (RES_W * RES_H * 3), f.fb,
                      RES_W * RES_H * 3);
        // the rollout's copy of the step's frame: a final frame is not one (phase B stores the env's next first frame)
        if (ROLL && !is_final_frame<PASS>(p, env_of())) {
            pg_bulk_store(p.roll.rgb + rollout_index(p, env_of()) * (RES_W * RES_H * 3), f.fb, RES_W * RES_H * 3);
            rollout_store_scalars(p, env_of());
        }
        pg_bulk_commit_and_wait();
    }
    PG_RENDER_PHASE(7);
#undef PG_RENDER_PHASE
}

// A paused env's consumer epilogue. There is one ring position per handle, so the ring moves on for every env: the
// newest slot s and its twin s + k get the frame the env is paused on, which is in slot s - 1 because every step
// (and pgb200_set_consumer_output, and set_state) writes every env's current slot. Its older frames stay (first = 0).
__device__ __forceinline__ void consumer_repeat_frame(const KParams &p, int env) {
    constexpr int kSlotVecs = 3 * RES_W * RES_H * 2 / 16;  // 16-byte words of one 16-bit frame
    const int kf = p.consumer_k, s = *p.consumer_slot_dev;
    uint4 *base = reinterpret_cast<uint4 *>(p.consumer) + (size_t)env * (2 * kf) * kSlotVecs;
    const uint4 *src = base + (size_t)((s - 1 + kf) % kf) * kSlotVecs;
    for (int w = (int)threadIdx.x; w < kSlotVecs; w += kRenderThreads) {
        const uint4 v = src[w];
        base[(size_t)s * kSlotVecs + w] = v;
        base[(size_t)(s + kf) * kSlotVecs + w] = v;
    }
}

// PASS 0: a plain step, one CTA per env of the launch. With final outputs (pgb200_get_final_outputs):
// PASS 1 (phase A), the same grid, but the frame of an env whose level ended is its final frame: it goes to
// final_rgb and skips the consumer epilogue, whose episode-start rule would read the previous step's first[env].
// PASS 2 (phase B), a fixed grid whose CTAs loop over the envs phase A listed, after their reset: the mbarrier is
// re-armed per env with alternating parity, and the bulk store's wait_group.read 0 has already released the frame.
// PAUSE (PASS 0 and 1, a handle with a pause mask): the CTA of an env paused in this step renders nothing; its rgb
// slot keeps the frame it is paused on, and the consumer ring and the rollout get that frame again
// (consumer_repeat_frame, rollout_copy_frame; the paused step's rew and first are 0).
// ROLL: the handle has a rollout (pgb200_get_rollout), which every frame of the step is also stored to. A separate
// instantiation, so that the render kernel of a handle without one keeps its registers and stack.
template <class G, int VIEW, int PASS = 0, bool PAUSE = false, bool ROLL = false>
__global__ void __launch_bounds__(kRenderThreads, RenderTune<G, VIEW>::kMinBlocks) render_kernel(KParams p) {
    static_assert(!(PAUSE && PASS == 2), "phase B's list never holds a paused env");
    using Frame = typename FrameFor<G, VIEW>::type;
    extern __shared__ __align__(128) unsigned char smem_raw[];
    Frame &f = *reinterpret_cast<Frame *>(smem_raw);
    if (PAUSE && p.paused[p.env_first + (int)blockIdx.x * p.env_step]) {
        if (p.consumer != nullptr && p.consumer_k > 1)
            consumer_repeat_frame(p, p.env_first + (int)blockIdx.x * p.env_step);
        if (ROLL)
            rollout_copy_frame(p, p.env_first + (int)blockIdx.x * p.env_step, (int)threadIdx.x, kRenderThreads);
        return;
    }
    if (threadIdx.x == 0)
        pg_mbar_init(&f.mbar, 1);
    __syncthreads();
    if (PASS == 2) {
        // the list entry is kept in shared memory and the count re-read each round
        __shared__ int list_env;
        for (unsigned i = 0;; i++) {
            const int j = (int)(blockIdx.x + i * gridDim.x);
            if (j >= (int)*p.reset_count)
                break;
            if (threadIdx.x == 0)
                list_env = p.reset_list[j];
            __syncthreads();
            render_env_frame<G, VIEW, PASS, ROLL>(p, f, [&] { return list_env; }, i & 1u);
            __syncthreads();
        }
        return;
    }
    render_env_frame<G, VIEW, PASS, ROLL>(p, f, [&] { return p.env_first + (int)blockIdx.x * p.env_step; }, 0);
}

// Game::observe without a step (set_state, vecgame.cpp:454-456): camera, then the frame kernels
template <class G>
__global__ void camera_kernel(KParams p) {
    using Frame = typename FrameFor<G>::type;
    if (threadIdx.x == 0 && blockIdx.x < (unsigned)p.env_count)
        env_observe<G, Frame>(p, p.env_first + (int)blockIdx.x * p.env_step);
}

// The same camera for the envs p.reset_list holds (set_state of a list of envs): block j takes entry j
template <class G>
__global__ void camera_list_kernel(KParams p) {
    using Frame = typename FrameFor<G>::type;
    if (threadIdx.x == 0 && blockIdx.x < *p.reset_count)
        env_observe<G, Frame>(p, p.reset_list[blockIdx.x]);
}
#endif

// the setup + render kernels' phases as plain loops (host debug harness; also documents the phase order). PASS and
// ROLL: see render_kernel; in pass 1 the frame of an env whose level ended goes to final_rgb, and skips the rollout.
template <class G, int VIEW, int PASS, bool ROLL>
void render_env_serial(const KParams &p, int env) {
    using Frame = typename FrameFor<G, VIEW>::type;
    using Setup = typename FrameFor<G, VIEW>::setup;
    using Shared = typename FrameFor<G, VIEW>::shared;
    static thread_local Frame *f = new Frame;
    static thread_local Setup *s = new Setup;
    // The device's record is a shared-memory slot that holds whatever its warp's previous env left in it. Here it is
    // poisoned before every frame, so that the parity suites fail if setup reads a field it has not written for this
    // frame, or if the render path depends on a stored byte that setup left unwritten.
    memset(static_cast<void *>(s), 0xA5, sizeof(Setup));
    env_setup_frame<G, Setup>(p, env, *s, 0, 1);
    env_store_frame<Setup>(p, env, *s);
    static_cast<Shared &>(*f) = *reinterpret_cast<const Shared *>(p.frame_setup + (size_t)env * p.frame_setup_stride);
    env_stage_tiles_serial<Frame>(p, *f);
    for (int w = 0; w < 4; w++) env_render_compose<G, Frame>(p, *f, w, 4, 0, 1);  // the device's row ownership, one lane per owner
    const bool final_frame = is_final_frame<PASS>(p, env);
    uint8_t *rgb = final_frame ? p.final_rgb : p.rgb;
    uint32_t *out = reinterpret_cast<uint32_t *>(rgb + (size_t)env * (RES_W * RES_H * 3));
    for (int g = 0; g < RES_W * RES_H / 4; g++) Raster<G, Frame>::pack_quad(f->fb + 4 * g, out + 3 * g);
    if (ROLL && !final_frame)
        rollout_copy_frame(p, env, 0, 1);
}

// The work counters of one launch slot (VecEnv keeps kMaxTickets of them, one per launch in flight). The logic phase
// clears the words its step uses (ticket_bytes) before its kernel, on the stream the launch's kernels follow.
struct alignas(32) TicketSlot {
    unsigned int logic;        // the logic kernel's ticket
    unsigned int reset_count;  // two-phase: the envs phase A put in reset_list
    unsigned int finish;       // two-phase: the finish kernel's ticket
    unsigned int look_count;   // level lookahead: the envs phase B put in look.list (the lookahead kernel's count[0])
    unsigned int look;         // level lookahead: the lookahead kernel's ticket (its count[1])
};

// The kernels a step runs, from the opt-ins the handle has (VecEnv::step_shape, once per step). A handle without an
// opt-in runs exactly the kernels it ran before the opt-in existed.
struct StepShape {
    bool init = false;           // the initial reset: the logic kernel's INIT instantiation, and no opt-in
    bool level_choice = false;   // next_level_seed: a one-phase step's logic kernel takes the caller's next level
    bool pause = false;          // pause mask
    bool final_outputs = false;  // final outputs: phase B renders again
    bool bank = false;           // level bank
    bool look = false;           // level lookahead: its kernel follows phase B
    bool roll = false;           // rollout: the render kernel's ROLL instantiation, and a cursor advance per step
    bool repeat = false;         // action repeat: the logic and finish kernels' REPEAT instantiations
    // A step in two phases: the logic kernel (phase A) lists the envs whose level ends, and the finish kernel (phase B)
    // resets them. Its logic kernel is one that steps always run (its stack frame and registers stay those of the
    // step, which must fit the push_obj / sub_step recursion).
    bool two_phase() const { return final_outputs || bank || look; }
    // the words of TicketSlot the step uses
    size_t ticket_bytes() const {
        return look ? offsetof(TicketSlot, look) + sizeof(unsigned int)
                    : two_phase() ? offsetof(TicketSlot, finish) + sizeof(unsigned int) : sizeof(unsigned int);
    }
};

struct LaunchCtx {
    Stream stream;
    Stream logic_stream;      // null, or a higher-priority stream the logic kernel goes to (then `link` orders render behind it)
    Event link;
    int max_logic_blocks;     // SM count x resident CTAs per SM
    int num_sms;              // SM count: sizes the machine-filling grids of a final-outputs step's phase B
    int render_smem_floor;    // dynamic shared memory requested per render CTA is at least this (co-residency knob)
    Event *tev;               // optional: 4 events (before logic, after it, after setup, after render) for kernel timing
    TicketSlot *ticket;       // this launch's slot
    Stream look_stream;       // level lookahead: the side stream the launch's lookahead kernel runs on, forked at
    Event look_fork;          // look_fork behind phase B (the runtime joins it back behind the launch's last work)
    int64_t *launch_counter;  // pgb200_kernel_launches: each phase adds the kernels it launches
};

// f(std::true_type{}) or f(std::false_type{}): one flag of a step's shape as a template argument of what f launches
template <class F>
void with_flag(bool flag, F &&f) {
    if (flag)
        f(std::true_type{});
    else
        f(std::false_type{});
}

#ifndef PG_HOSTSIM
// `bytes` of dynamic shared memory for kernel K, with K's opt-in limit raised to them where a launch first needs it
template <auto K>
int dynamic_smem(int bytes) {
    // the attribute is per device: remember what each device of this process was given
    static int attr_set[64] = {};
    int dev = 0;
    CUDA_CHECK(cudaGetDevice(&dev));
    int &have = attr_set[dev & 63];
    if (have < bytes) {
        CUDA_CHECK(cudaFuncSetAttribute(K, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
        have = bytes;
    }
    return bytes;
}

// grid of the persistent logic and finish kernels: one warp per env, at most what the machine holds at once
static inline int logic_grid(const KParams &p, const LaunchCtx &lc) {
    const int blocks = (p.env_count + kLogicEnvsPerBlock - 1) / kLogicEnvsPerBlock;
    return blocks < lc.max_logic_blocks ? blocks : lc.max_logic_blocks;
}
#endif

// The phases of a step. Each turns the flags of the shape it depends on into template arguments, launches its
// kernels on the launch's stream or, in the host debug build, runs the same per-env code as a loop over the launch's
// envs or over the reset list, and counts one launch per kernel.

// logic: clears the words of the launch's ticket slot the step uses, then runs the logic kernel over the launch's envs.
// A two-phase step stays on lc.stream: a priority-split logic stream would let the next launch that shares this ticket
// slot clear it under phase B. A one-phase step's logic kernel may go to that stream (PGB200_PRIORITY_SPLIT).
template <class G, bool INIT, bool LEVEL_CHOICE, bool FINAL, bool PAUSE, bool REPEAT>
void logic_kernels(const KParams &p, const LaunchCtx &lc, size_t ticket_bytes) {
#ifndef PG_HOSTSIM
    const cudaStream_t ls = !FINAL && lc.logic_stream ? lc.logic_stream : lc.stream;
    CUDA_CHECK(cudaMemsetAsync(lc.ticket, 0, ticket_bytes, ls));
    if (lc.tev)
        CUDA_CHECK(cudaEventRecord(lc.tev[0], ls));
    logic_kernel<G, INIT, LEVEL_CHOICE, FINAL, PAUSE, REPEAT><<<logic_grid(p, lc), kLogicThreads, 0, ls>>>(p, &lc.ticket->logic);
    CUDA_CHECK(cudaGetLastError());
    if (ls != lc.stream) {
        CUDA_CHECK(cudaEventRecord(lc.link, ls));
        CUDA_CHECK(cudaStreamWaitEvent(lc.stream, lc.link, 0));
    }
#else
    using Frame = typename FrameFor<G>::type;
    memset(lc.ticket, 0, ticket_bytes);
    for (int i = 0; i < p.env_count; i++) env_logic<G, Frame, INIT, LEVEL_CHOICE, FINAL, PAUSE, REPEAT>(p, p.env_first + i * p.env_step);
#endif
    (*lc.launch_counter) += 1;
}

// INIT, or a step: FINAL (phase A) when it has two phases, LEVEL_CHOICE only when it has one, PAUSE with a pause mask,
// REPEAT with action repeat
template <class G>
void logic_phase(const KParams &p, const LaunchCtx &lc, const StepShape &s) {
    if (s.init)
        return logic_kernels<G, true, false, false, false, false>(p, lc, s.ticket_bytes());
    with_flag(s.repeat, [&](auto repeat) {
        with_flag(s.pause, [&](auto pause) {
            with_flag(s.two_phase(), [&](auto final) {
                if constexpr (final)
                    logic_kernels<G, false, false, true, pause, repeat>(p, lc, s.ticket_bytes());
                else
                    with_flag(s.level_choice,
                              [&](auto choice) { logic_kernels<G, false, choice, false, pause, repeat>(p, lc, s.ticket_bytes()); });
            });
        });
    });
}

// finish: phase B's resets, the finish kernel over the envs phase A listed. BANK: they copy their levels from the
// bank where it holds them. LOOK: or from their lookahead slots, and list the envs whose next level is to be generated.
// REPEAT: their rew adds the reset's reward to phase A's sum.
template <class G>
void finish_phase(const KParams &p, const LaunchCtx &lc, const StepShape &s) {
    with_flag(s.bank, [&](auto bank) {
        with_flag(s.look, [&](auto look) {
            with_flag(s.repeat, [&](auto repeat) {
#ifndef PG_HOSTSIM
                finish_kernel<G, bank, look, repeat><<<logic_grid(p, lc), kLogicThreads, 0, lc.stream>>>(p, &lc.ticket->finish);
                CUDA_CHECK(cudaGetLastError());
#else
                using Frame = typename FrameFor<G>::type;
                for (unsigned int j = 0; j < *p.reset_count; j++) env_finish_logic<G, Frame, bank, look, repeat>(p, p.reset_list[j]);
#endif
            });
        });
    });
    (*lc.launch_counter) += 1;
}

// lookahead: the lookahead kernel over the envs phase B listed, on the launch's side stream forked here, so that it
// runs beside the frames phase (the runtime joins it back). The host debug build runs it in place, before the frames.
template <class G>
void lookahead_phase(const KParams &p, const LaunchCtx &lc) {
#ifndef PG_HOSTSIM
    CUDA_CHECK(cudaEventRecord(lc.look_fork, lc.stream));
    CUDA_CHECK(cudaStreamWaitEvent(lc.look_stream, lc.look_fork, 0));
    const int blocks = (p.look.stage_warps + kLogicEnvsPerBlock - 1) / kLogicEnvsPerBlock;
    lookahead_kernel<G><<<blocks, kLogicThreads, 0, lc.look_stream>>>(p, p.look.count);
    CUDA_CHECK(cudaGetLastError());
#else
    for (unsigned int j = 0; j < *p.look.count; j++) lookahead_generate<G>(p, (int)j, p.look.stage);
#endif
    (*lc.launch_counter) += 1;
}

// frames: the setup kernel, then the render kernel of pass PASS, between kernel-timing events 1 to 3 (the runtime
// gives a step with final outputs none). PASS 0 and 1 cover the launch's envs, and PAUSE leaves the paused ones'
// frames as they are. PASS 2 covers the envs phase A listed: its grids are fixed (machine-filling) and read the
// list's count on the device, so nothing waits for the host and the step stays capturable. ROLL: the render kernel
// also stores every frame to the rollout.
template <class G, int VIEW, int PASS, bool PAUSE, bool ROLL>
void frames_kernels(const KParams &p, const LaunchCtx &lc) {
    constexpr bool LIST = PASS == 2;
#ifndef PG_HOSTSIM
    using Frame = typename FrameFor<G, VIEW>::type;
    const int setup_smem = dynamic_smem<setup_kernel<G, VIEW, LIST, PAUSE>>(SetupTune<G, VIEW>::kSmemBytes);
    const int render_smem = dynamic_smem<render_kernel<G, VIEW, PASS, PAUSE, ROLL>>(
        (int)sizeof(Frame) > lc.render_smem_floor ? (int)sizeof(Frame) : lc.render_smem_floor);
    int setup_blocks = (p.env_count + kSetupThreads / 32 - 1) / (kSetupThreads / 32);
    int render_blocks = p.env_count;
    if (LIST) {
        const int setup_fit = lc.num_sms * SetupTune<G, VIEW>::kMinBlocks, render_fit = lc.num_sms * RenderTune<G, VIEW>::kMinBlocks;
        setup_blocks = setup_blocks < setup_fit ? setup_blocks : setup_fit;
        render_blocks = render_blocks < render_fit ? render_blocks : render_fit;
    }
    if (lc.tev)
        CUDA_CHECK(cudaEventRecord(lc.tev[1], lc.stream));
    setup_kernel<G, VIEW, LIST, PAUSE><<<setup_blocks, kSetupThreads, setup_smem, lc.stream>>>(p);
    if (lc.tev)
        CUDA_CHECK(cudaEventRecord(lc.tev[2], lc.stream));
    render_kernel<G, VIEW, PASS, PAUSE, ROLL><<<render_blocks, kRenderThreads, render_smem, lc.stream>>>(p);
    if (lc.tev)
        CUDA_CHECK(cudaEventRecord(lc.tev[3], lc.stream));
    CUDA_CHECK(cudaGetLastError());
#else
    (void)lc;
    if (LIST) {
        for (unsigned int j = 0; j < *p.reset_count; j++) render_env_serial<G, VIEW, PASS, ROLL>(p, p.reset_list[j]);
    } else {
        for (int i = 0; i < p.env_count; i++) {
            const int env = p.env_first + i * p.env_step;
            if (!(PAUSE && p.paused[env]))
                render_env_serial<G, VIEW, PASS, ROLL>(p, env);
            else if (ROLL)
                rollout_copy_frame(p, env, 0, 1);
        }
    }
#endif
    (*lc.launch_counter) += 2;
}

template <class G, int VIEW, int PASS>
void frames_phase(const KParams &p, const LaunchCtx &lc, const StepShape &s) {
    with_flag(s.roll, [&](auto roll) {
        if constexpr (PASS == 2)  // phase B's list never holds a paused env
            frames_kernels<G, VIEW, PASS, false, roll>(p, lc);
        else
            with_flag(s.pause, [&](auto pause) { frames_kernels<G, VIEW, PASS, pause, roll>(p, lc); });
    });
}

// One (game, env chunk) launch of a step (or of the initial reset), as its phases:
//   initial reset, one-phase step                    logic, frames(0)
//   two-phase step without final outputs             logic (phase A), finish [, lookahead], frames(0)
//   final outputs (with or without bank, lookahead)  logic (phase A), frames(1), finish [, lookahead], frames(2)
// The lookahead phase (level lookahead) runs beside the frames that follow it.
// A final-outputs step's phase A renders the final frames of the envs whose level ends, to final_rgb; phase B renders
// the first frames of their next levels. Without final outputs, phase A's level_end goes to the handle's
// bank_level_end. The lists' counts are words of the launch's ticket slot.
template <class G, int VIEW>
void launch_step(const KParams &p, const LaunchCtx &lc, const StepShape &s) {
    if (p.env_count <= 0)
        return;
    if (!s.two_phase()) {
        logic_phase<G>(p, lc, s);
        frames_phase<G, VIEW, 0>(p, lc, s);
        return;
    }
    KParams q = p;  // what the phases of a two-phase step see
    q.reset_count = &lc.ticket->reset_count;
    q.look.count = &lc.ticket->look_count;
    if (!s.final_outputs)
        q.level_end = p.bank_level_end;
    logic_phase<G>(q, lc, s);
    if (s.final_outputs)
        frames_phase<G, VIEW, 1>(q, lc, s);
    finish_phase<G>(q, lc, s);
    if (s.look)
        lookahead_phase<G>(q, lc);
    if (s.final_outputs)
        frames_phase<G, VIEW, 2>(q, lc, s);
    else
        frames_phase<G, VIEW, 0>(p, lc, s);
}

// An observation without a step (set_state, the consumer output's first frame): the camera, then the frames of a step
// without pause mask or rollout, which it leaves alone. pgb200_kernel_launches counts the two frame kernels.
template <class G, int VIEW>
void launch_observe_only(const KParams &p, const LaunchCtx &lc) {
    if (p.env_count <= 0)
        return;
#ifndef PG_HOSTSIM
    camera_kernel<G><<<p.env_count, 32, 0, lc.stream>>>(p);
    CUDA_CHECK(cudaGetLastError());
#else
    using Frame = typename FrameFor<G>::type;
    for (int i = 0; i < p.env_count; i++) env_observe<G, Frame>(p, p.env_first + i * p.env_step);
#endif
    frames_phase<G, VIEW, 0>(p, lc, StepShape{});
}

// launch_observe_only for the p.env_count envs p.reset_list holds (*p.reset_count on the device), distinct envs of the
// launch's game: the list camera, then the frames of phase B of a step without rollout. Phase B's render pass differs
// from pass 0 only in taking its envs from the list, so the listed envs get what launch_observe_only gives them (rgb,
// rew, first, the infos and the consumer ring's current slot) and the rollout is left alone. Counted as launch_observe_only.
template <class G, int VIEW>
void launch_observe_list(const KParams &p, const LaunchCtx &lc) {
    if (p.env_count <= 0)
        return;
#ifndef PG_HOSTSIM
    camera_list_kernel<G><<<p.env_count, 32, 0, lc.stream>>>(p);
    CUDA_CHECK(cudaGetLastError());
#else
    using Frame = typename FrameFor<G>::type;
    for (unsigned int j = 0; j < *p.reset_count; j++) env_observe<G, Frame>(p, p.reset_list[j]);
#endif
    frames_phase<G, VIEW, 2>(p, lc, StepShape{});
}

// Generates p.bank's levels [0, count) of the launch's game: `warps` warps, each with bank_stage_bytes(p) of `stage`.
// Counted as a launch in the device build only.
template <class G>
void launch_bank_build(const KParams &p, const LaunchCtx &lc, unsigned char *stage, int warps, int count) {
    if (count <= 0)
        return;
#ifndef PG_HOSTSIM
    const int blocks = (warps + kLogicEnvsPerBlock - 1) / kLogicEnvsPerBlock;
    bank_build_kernel<G><<<blocks, kLogicThreads, 0, lc.stream>>>(p, stage, count, warps);
    CUDA_CHECK(cudaGetLastError());
    (*lc.launch_counter) += 1;
#else
    (void)lc;
    (void)warps;
    for (int item = 0; item < count; item++)
        bank_generate_level<G>(p, p.bank, p.bank.seeds[item], [&] { return p.bank.slots + (size_t)item * p.bank.slot_bytes; }, stage);
#endif
}

// Level lookahead's bulk fill of the launch's envs: every env's next level predicted, then the listed ones generated
// by p.look.stage_warps warps with staging at p.look.stage, on the launch's stream. p.look.count: the lookahead words
// of a ticket slot, zero. Counted as two launches in the device build only.
template <class G>
void launch_lookahead_fill(const KParams &p, const LaunchCtx &lc) {
    if (p.env_count <= 0)
        return;
#ifndef PG_HOSTSIM
    lookahead_predict_kernel<G><<<(p.env_count + kLogicEnvsPerBlock - 1) / kLogicEnvsPerBlock, kLogicThreads, 0, lc.stream>>>(p);
    CUDA_CHECK(cudaGetLastError());
    const int blocks = (p.look.stage_warps + kLogicEnvsPerBlock - 1) / kLogicEnvsPerBlock;
    lookahead_kernel<G><<<blocks, kLogicThreads, 0, lc.stream>>>(p, p.look.count);
    CUDA_CHECK(cudaGetLastError());
    (*lc.launch_counter) += 2;
#else
    (void)lc;
    for (int i = 0; i < p.env_count; i++) lookahead_predict(p, p.env_first + i * p.env_step, p.bank.slots != nullptr);
    for (unsigned int j = 0; j < *p.look.count; j++) lookahead_generate<G>(p, (int)j, p.look.stage);
#endif
}

struct GameVTable {
    const char *name;
    int id;
    int ent_cap, grid_cap, scratch_words;
    int rot_records;  // rotated-sprite / span records per env (global)
    int blit_records; // blit list capacity per env (global)
    // [0] = the game's usual view, [1] = the whole-world view of center_agent = false (step[1] null: the game has none)
    int setup_bytes[2];   // sizeof(FrameSharedT): the global record the setup kernel stores and the render kernel stages
    int cell_records[2];  // cells of the largest visible window (capacity for general cell blits)
    int frame_bytes[2];   // shared memory of one render CTA
    int render_ctas_per_sm[2];  // residency the render kernel is compiled for
    void (*step[2])(const KParams &, const LaunchCtx &, const StepShape &);  // a step or the initial reset (launch_step)
    void (*observe_only[2])(const KParams &, const LaunchCtx &);
    void (*observe_list[2])(const KParams &, const LaunchCtx &);
    void (*bank_build)(const KParams &, const LaunchCtx &, unsigned char *, int, int);
    void (*lookahead_fill)(const KParams &, const LaunchCtx &);
    int persist_scratch_first, persist_scratch_words;  // G::PERSIST_SCRATCH_FIRST / _WORDS
};

template <class G, int VIEW>
void fill_view(GameVTable &vt, int slot) {
    using F = FrameFor<G, VIEW>;
    vt.setup_bytes[slot] = (int)sizeof(typename F::shared);
    vt.cell_records[slot] = F::type::kMaxCells1D * F::type::kMaxCells1D;
    vt.frame_bytes[slot] = (int)sizeof(typename F::type);
#ifndef PG_HOSTSIM
    vt.render_ctas_per_sm[slot] = RenderTune<G, VIEW>::kMinBlocks;
#else
    vt.render_ctas_per_sm[slot] = 0;
#endif
    vt.step[slot] = &launch_step<G, VIEW>;
    vt.observe_only[slot] = &launch_observe_only<G, VIEW>;
    vt.observe_list[slot] = &launch_observe_list<G, VIEW>;
}

template <class G>
GameVTable make_vtable(int id) {
    GameVTable vt{};
    vt.name = G::NAME;
    vt.id = id;
    vt.ent_cap = G::ENT_CAP;
    vt.grid_cap = G::GRID_CAP;
    vt.scratch_words = G::SCRATCH_WORDS;
    vt.persist_scratch_first = G::PERSIST_SCRATCH_FIRST;
    vt.persist_scratch_words = G::PERSIST_SCRATCH_WORDS;
    vt.bank_build = &launch_bank_build<G>;
    vt.lookahead_fill = &launch_lookahead_fill<G>;
    vt.rot_records = FrameFor<G>::type::kMaxRot;
    vt.blit_records = FrameFor<G>::type::kMaxList;
    fill_view<G, G::MAX_VIEW_CELLS>(vt, 0);
    if constexpr (G::FULL_VIEW_CELLS > G::MAX_VIEW_CELLS)
        fill_view<G, G::FULL_VIEW_CELLS>(vt, 1);
    return vt;
}

}  // namespace pg
