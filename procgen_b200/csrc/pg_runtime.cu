// libprocgen_b200.so — host runtime + CUDA kernels + the C ABI of include/procgen_b200.h.
//
// Replaces the reference's vector runtime (vecgame.cpp: N Game objects + worker-thread pool behind
// one mutex and two condvars) with: all env state resident in HBM, one CTA per env, one
// asynchronous kernel launch per act() on a private stream, and observe() = stream wait.
//
// Build modes: nvcc (product, sm_90a).  With -DPG_HOSTSIM the same file builds with g++ into the
// CPU debug harness used ONLY by tests/ (every kernel becomes a plain loop); that build reports
// pgb200_is_device_build() == 0 and the Python package refuses to load it. The two builds part ways
// once for memory, copies and streams (the build seam below); past it they differ only where they do
// different work: the device-only kernels, a step's stream fork / join and copies, device setup,
// page-locking the caller's observations, and the entry points the host build refuses.
//
// A handle (VecEnv) owns every device array, pinned buffer, stream and event it creates: each is
// registered with it when it is made, and ~VecEnv releases them all.
#include <dlfcn.h>
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <atomic>
#include <exception>
#include <memory>
#include <mutex>
#include <random>
#include <stdexcept>
#include <string>
#include <thread>
#include <vector>

#include "../../include/procgen_b200.h"
#include "pg_asset_tables.h"
#include "pg_launch.cuh"
#include "games/bigfish.cuh"
#include "games/bossfight.cuh"
#include "games/dodgeball.cuh"
#include "games/caveflyer.cuh"
#include "games/chaser.cuh"
#include "games/climber.cuh"
#include "games/coinrun.cuh"
#include "games/fruitbot.cuh"
#include "games/heist.cuh"
#include "games/jumper.cuh"
#include "games/leaper.cuh"
#include "games/maze.cuh"
#include "games/miner.cuh"
#include "games/ninja.cuh"
#include "games/plunder.cuh"
#include "games/starpilot.cuh"
#include "pg_state_io.h"

namespace pg {
const GameVTable *pg_vtable_bigfish();
const GameVTable *pg_vtable_bossfight();
const GameVTable *pg_vtable_dodgeball();
const GameVTable *pg_vtable_caveflyer();
const GameVTable *pg_vtable_chaser();
const GameVTable *pg_vtable_climber();
const GameVTable *pg_vtable_coinrun();
const GameVTable *pg_vtable_fruitbot();
const GameVTable *pg_vtable_heist();
const GameVTable *pg_vtable_jumper();
const GameVTable *pg_vtable_leaper();
const GameVTable *pg_vtable_maze();
const GameVTable *pg_vtable_miner();
const GameVTable *pg_vtable_ninja();
const GameVTable *pg_vtable_plunder();
const GameVTable *pg_vtable_starpilot();
}  // namespace pg

using namespace pg;

// ================================================================= build seam
// What the runtime asks of CUDA, once per build. The host debug build keeps "device" memory on the heap,
// copies with memcpy and finishes every launch before it returns: it has nothing to wait for and never captures.
#ifndef PG_HOSTSIM
#include <cuda_fp16.h>
#include <cuda_runtime.h>

static constexpr int kDeviceBuild = 1;
static inline void set_current_device(int device) { CUDA_CHECK(cudaSetDevice(device)); }
// device memory, left as it is
static inline void *dev_malloc(size_t bytes) {
    void *ptr = nullptr;
    CUDA_CHECK(cudaMalloc(&ptr, bytes));
    return ptr;
}
static inline void dev_free(void *ptr) { cudaFree(ptr); }
// device memory, or null when the device cannot provide it
static inline void *dev_try_malloc(size_t bytes) {
    void *ptr = nullptr;
    if (cudaMalloc(&ptr, bytes) != cudaSuccess) {
        cudaGetLastError();
        return nullptr;
    }
    return ptr;
}
static inline void *pinned_alloc(size_t bytes) {
    void *ptr = nullptr;
    CUDA_CHECK(cudaHostAlloc(&ptr, bytes, cudaHostAllocDefault));
    return ptr;
}
static inline void pinned_free(void *ptr) { cudaFreeHost(ptr); }
static inline void host_unregister(void *ptr) { cudaHostUnregister(ptr); }
static inline void stream_destroy(Stream s) { cudaStreamDestroy(s); }
static inline void event_destroy(Event e) { cudaEventDestroy(e); }
// on the legacy default stream, complete when they return
static inline void dev_memset(void *dst, int value, size_t bytes) { CUDA_CHECK(cudaMemset(dst, value, bytes)); }
// `rows` runs of `bytes` bytes, `pitch` bytes apart
static inline void memset_strided(void *dst, int value, size_t bytes, size_t pitch, size_t rows) {
    if (rows)
        CUDA_CHECK(cudaMemset2D(dst, pitch, value, bytes, rows));
}
static inline void copy_to_dev(void *dst, const void *src, size_t bytes) { CUDA_CHECK(cudaMemcpy(dst, src, bytes, cudaMemcpyHostToDevice)); }
static inline void copy_from_dev(void *dst, const void *src, size_t bytes) { CUDA_CHECK(cudaMemcpy(dst, src, bytes, cudaMemcpyDeviceToHost)); }
// on stream s, behind the work issued there before
static inline void copy_to_dev_async(void *dst, const void *src, size_t bytes, Stream s) {
    CUDA_CHECK(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, s));
}
static inline void copy_from_dev_async(void *dst, const void *src, size_t bytes, Stream s) {
    CUDA_CHECK(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, s));
}
static inline void copy_dev_async(void *dst, const void *src, size_t bytes, Stream s) {
    CUDA_CHECK(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToDevice, s));
}
static inline void memset_async(void *dst, int value, size_t bytes, Stream s) { CUDA_CHECK(cudaMemsetAsync(dst, value, bytes, s)); }
static inline void stream_sync(Stream s) { CUDA_CHECK(cudaStreamSynchronize(s)); }
static inline void device_sync() { CUDA_CHECK(cudaDeviceSynchronize()); }
// Whether `s` is capturing a CUDA graph. Querying the legacy stream while another stream captures in a
// non-relaxed mode reports cudaErrorStreamCaptureImplicit: work there would join that capture, so it counts.
static inline bool stream_capturing(Stream s) {
    cudaStreamCaptureStatus st = cudaStreamCaptureStatusNone;
    const cudaError_t e = cudaStreamIsCapturing(s, &st);
    if (e == cudaErrorStreamCaptureImplicit) {
        cudaGetLastError();
        return true;
    }
    CUDA_CHECK(e);
    return st != cudaStreamCaptureStatusNone;
}
#else
static constexpr int kDeviceBuild = 0;
static inline void set_current_device(int) {}
static inline void *dev_malloc(size_t bytes) { return calloc(bytes, 1); }
static inline void dev_free(void *ptr) { free(ptr); }
static inline void *dev_try_malloc(size_t bytes) { return calloc(bytes, 1); }
static inline void *pinned_alloc(size_t bytes) { return malloc(bytes); }
static inline void pinned_free(void *ptr) { free(ptr); }
static inline void host_unregister(void *) {}
static inline void stream_destroy(Stream) {}
static inline void event_destroy(Event) {}
static inline void dev_memset(void *dst, int value, size_t bytes) { memset(dst, value, bytes); }
static inline void memset_strided(void *dst, int value, size_t bytes, size_t pitch, size_t rows) {
    for (size_t r = 0; r < rows; r++) memset((unsigned char *)dst + r * pitch, value, bytes);
}
static inline void copy_to_dev(void *dst, const void *src, size_t bytes) { memcpy(dst, src, bytes); }
static inline void copy_from_dev(void *dst, const void *src, size_t bytes) { memcpy(dst, src, bytes); }
static inline void copy_to_dev_async(void *dst, const void *src, size_t bytes, Stream) { memcpy(dst, src, bytes); }
static inline void copy_from_dev_async(void *dst, const void *src, size_t bytes, Stream) { memcpy(dst, src, bytes); }
static inline void copy_dev_async(void *dst, const void *src, size_t bytes, Stream) { memcpy(dst, src, bytes); }
static inline void memset_async(void *dst, int value, size_t bytes, Stream) { memset(dst, value, bytes); }
static inline void stream_sync(Stream) {}
static inline void device_sync() {}
static inline bool stream_capturing(Stream) { return false; }
#endif

// ================================================================= option parsing (vecoptions.cpp)
namespace {

struct OptParser {
    std::vector<libenv_option> opts;
    explicit OptParser(const libenv_options &o) : opts(o.items, o.items + o.count) {}
    bool find(const std::string &name, libenv_dtype dtype, libenv_option *out) {
        for (size_t i = 0; i < opts.size(); i++) {
            if (name == std::string(opts[i].name)) {
                if (opts[i].dtype != dtype)
                    pg_fatal("invalid dtype for option %s\n", name.c_str());
                *out = opts[i];
                opts.erase(opts.begin() + i);
                return true;
            }
        }
        return false;
    }
    void consume_string(const std::string &name, std::string *v) {
        libenv_option o;
        if (find(name, LIBENV_DTYPE_UINT8, &o))
            *v = std::string((char *)o.data, o.count);
    }
    void consume_int(const std::string &name, int32_t *v) {
        libenv_option o;
        if (find(name, LIBENV_DTYPE_INT32, &o))
            *v = *(int32_t *)o.data;
    }
    void consume_bool(const std::string &name, bool *v) {
        libenv_option o;
        if (find(name, LIBENV_DTYPE_UINT8, &o)) {
            uint8_t b = *(uint8_t *)o.data;
            pg_fassert(b == 0 || b == 1);
            *v = (bool)b;
        }
    }
    void ensure_empty() {
        if (!opts.empty())
            pg_fatal("unused options found, first unused option: %s\n", opts[0].name);
    }
};

std::vector<std::string> split(std::string s, const std::string &delim) {
    std::vector<std::string> out;
    size_t pos;
    while ((pos = s.find(delim)) != std::string::npos) {
        out.push_back(s.substr(0, pos));
        s.erase(0, pos + delim.length());
    }
    out.push_back(s);
    return out;
}

const GameVTable *find_game(const std::string &name) {
    // one entry per games_tu/tu_<game>.cu
    static const GameVTable *const table[] = {
        pg_vtable_bigfish(),
        pg_vtable_bossfight(),
        pg_vtable_dodgeball(),
        pg_vtable_caveflyer(),
        pg_vtable_chaser(),
        pg_vtable_climber(),
        pg_vtable_coinrun(),
        pg_vtable_fruitbot(),
        pg_vtable_heist(),
        pg_vtable_jumper(),
        pg_vtable_leaper(),
        pg_vtable_maze(),
        pg_vtable_miner(),
        pg_vtable_ninja(),
        pg_vtable_plunder(),
        pg_vtable_starpilot(),
    };
    for (const GameVTable *g : table)
        if (name == g->name)
            return g;
    return nullptr;
}

// The bank's slot layout of game g (pg_bank.cuh), for levels generated with `options`: int32 usable, int32 key (16 B) |
// EnvHdr | Entity[ENT_CAP] | grid[GRID_CAP] | MT19937 | persistent scratch. Bank slots and lookahead slots share it.
LevelBank slot_layout(const GameVTable *g, const Options &options) {
    LevelBank b{};
    b.ents_off = BANK_SLOT_HEAD + (int)sizeof(EnvHdr);
    b.grid_off = b.ents_off + g->ent_cap * (int)sizeof(Entity);
    b.rng_off = b.grid_off + ((g->grid_cap * (int)sizeof(int16_t) + 15) & ~15);
    b.scratch_off = b.rng_off + (int)sizeof(MT19937);
    b.slot_bytes = b.scratch_off + ((g->persist_scratch_words * (int)sizeof(int32_t) + 15) & ~15);
    b.options = options;
    return b;
}

// vecgame.cpp:156-167: system-independent hash of the game name
static int32_t fnv1a(const char *str) {
    uint32_t hash = 0x811c9dc5u;
    for (const char *c = str; *c; c++) {
        hash ^= (uint8_t)*c;
        hash *= 0x1000193u;
    }
    return (int32_t)hash;
}

// ================================================================= device-only kernels
#ifndef PG_HOSTSIM
// the pre-scaled tile table: one CTA per (sprite slot, tw, th)
__global__ void tile_table_kernel(const SpriteDesc *sprites, const uint32_t *index, uint32_t *texels, const uint32_t *atlas) {
    const int slot = (int)blockIdx.x / TILE_VARIANTS, v = (int)blockIdx.x % TILE_VARIANTS;
    tile_table_fill(sprites, index, texels, atlas, slot, v / MAX_TILE_DIM + 1, v % MAX_TILE_DIM + 1, (int)threadIdx.x, (int)blockDim.x);
}

// (16-bit float)(v / 255.f) for v = 0..255: IEEE fp32 division, then round-to-nearest-even
__global__ void consumer_lut_kernel(uint16_t *lut, int bf16) {
    const int v = (int)threadIdx.x;
    const float x = __fdiv_rn((float)v, 255.0f);
    if (bf16) {
        const uint32_t u = __float_as_uint(x);
        lut[v] = (uint16_t)((u + 0x7fffu + ((u >> 16) & 1u)) >> 16);
    } else {
        lut[v] = __half_as_ushort(__float2half_rn(x));
    }
}

// The ring position of the coming step (the consumer output's, the rollout's), advanced on the device so that a step
// captured in a CUDA graph moves it on at every replay (a kernel argument would be frozen at capture)
__global__ void ring_advance_kernel(int32_t *slot, int k) { *slot = (*slot + 1) % k; }

// State transfers, one warp per listed env. The headers of envs[0, count), which size the envs' packed records
__global__ void __launch_bounds__(128) state_headers_kernel(const EnvHdr *hdr, const int32_t *envs, int count, EnvHdr *out) {
    const int i = (int)((blockIdx.x * blockDim.x + threadIdx.x) >> 5);
    if (i < count)
        bank_copy_vecs(out + i, hdr + envs[i], (int)sizeof(EnvHdr));
}

// The packed records of slots[0, count) at recs: gathered from the envs (STORE false) or scattered into them
template <bool STORE>
__global__ void __launch_bounds__(128) state_records_kernel(KParams p, const StateSlot *slots, int count, unsigned char *recs) {
    const int i = (int)((blockIdx.x * blockDim.x + threadIdx.x) >> 5);
    if (i < count)
        state_move<STORE>(p, slots[i], recs + slots[i].offset);
}

// Snapshot slots (pgb200_apply_snapshots): the saves, one warp per slot, then the loads, one warp per env
__global__ void __launch_bounds__(128) snapshot_save_kernel(KParams p, SnapshotStore st) {
    const int s = (int)((blockIdx.x * blockDim.x + threadIdx.x) >> 5);
    if (s < st.count)
        snapshot_save(p, st, s);
}

__global__ void __launch_bounds__(128) snapshot_load_kernel(KParams p, SnapshotStore st) {
    const int env = (int)((blockIdx.x * blockDim.x + threadIdx.x) >> 5);
    if (env < st.num_envs)
        snapshot_load(p, st, env);
}
#endif

// ================================================================= VecEnv (VecGame, vecgame.h)
struct VecEnv {
    int num_envs = 0;
    int device = -1;
    std::vector<const GameVTable *> games;  // joint games, env n <-> games[n % size] (vecgame.cpp:310)
    std::vector<int> view;                  // per game: 0 = its usual view, 1 = the whole-world view (center_agent = false)
    std::vector<libenv_tensortype> observation_types, action_types, info_types;
    int num_actions = -1;

    KParams base{};                  // common launch parameters (a launch's own: game_params and its env range)
    std::vector<GameAssets *> d_assets;  // per joint game
    int32_t *d_action = nullptr;
    // The opt-in per-env arrays live in `base`, allocated by the first request for them (opt_in_array):
    // next_level_seed by pgb200_get_next_level_seeds; final_rgb and level_end by pgb200_get_final_outputs;
    // pause (the caller's mask, d_pause) and paused (what the logic kernel recorded of it for the step's later
    // kernels) by pgb200_get_pause_mask; bank_level_end by the first pgb200_build_level_bank. reset_list, the
    // pending-reset list of a two-phase step, by whichever of final outputs and the bank comes first. The rollout
    // (base.roll) by the first pgb200_get_rollout. The caller's repeat counts (d_repeat, base.repeat) by the first
    // pgb200_get_action_repeat.
    uint8_t *d_pause = nullptr;
    int32_t *d_repeat = nullptr;
    // allocated by the first pgb200_build_level_bank: bank_capacity slots per game of the list, sized by the game
    // (banks[g], one allocation at base.bank.slots), the sorted seed list they share and its length on the device
    std::vector<LevelBank> banks;
    int32_t *d_bank_seeds = nullptr, *d_bank_count = nullptr;
    int bank_capacity = 0;
    int bank_levels = 0;
    int64_t bank_bytes = 0;
    // allocated by pgb200_enable_level_lookahead: one slot per env in the bank's layout of its game (looks[g], one
    // allocation at base.look.slot.slots), the list the finish kernels fill and its per-step staging: look_warps warps
    // per side stream, one side stream (look_side, forked at look_fork and joined at look_join) per auxiliary stream
    std::vector<LevelLookahead> looks;
    int look_warps = 0;
    size_t look_stage_bytes = 0;             // per side stream
    unsigned long long *d_look_served = nullptr;
    int64_t look_bytes = 0;
    Stream look_side[PG_AUX_STREAMS] = {};
    Event look_fork[PG_AUX_STREAMS] = {}, look_join[PG_AUX_STREAMS] = {};
    bool initial_reset_done = false;
    int64_t launches = 0;
    host::ConstGameFields const_fields;  // options Game::serialize writes but no kernel reads

    // everything the handle allocates or creates, registered as it is made (alloc, alloc_pinned, own, opt_in_array)
    // and released by ~VecEnv
    std::vector<void *> owned_dev, owned_pinned;
    std::vector<Stream> owned_streams;
    std::vector<Event> owned_events;

    Stream stream = nullptr;  // where the handle's work goes: own_stream, or the caller's (pgb200_set_stream)
    Stream own_stream = nullptr;
    static constexpr int kAuxStreams = PG_AUX_STREAMS;
    Stream aux[kAuxStreams] = {};
    // PGB200_PRIORITY_SPLIT=1: logic kernels go to high-priority twins of the auxiliary streams so
    // their (small) blocks are dispatched ahead of the render CTAs queued by other chunks
    bool priority_split = false;
    Stream aux_hi[kAuxStreams] = {};
    Event ev_link[kAuxStreams] = {};
    Event ev_fork = nullptr;
    Event ev_join[kAuxStreams] = {};
    // optional per-launch kernel timing (pgb200_kernel_timing_begin/end): a pool of event quadruples
    std::vector<Event> tev_pool;
    std::vector<int> tev_envs;   // env count of each timed launch
    size_t tev_used = 0;
    bool timing = false;
    static constexpr int kChunks = PG_STEP_CHUNKS;
    int force_chunks = 0;            // measurement knobs (pgb200_set_launch_shape)
    bool serialize_launches = false;
    static constexpr int kMaxTickets = 64;   // launch slots in flight
    TicketSlot *d_tickets = nullptr;
    int max_logic_blocks = 1;        // logic blocks the device holds at once (device setup); the host build runs one env at a time
    int num_sms = 1;
    int render_smem_floor = 0;
    // host-buffer (libenv) mode
    // peer mirror (config 5, SURVEY §8e): when set, every launch's frames are also copied into
    // these buffers (another GPU's memory, mapped through NVLink) right behind its render kernel
    uint8_t *mirror[2] = {nullptr, nullptr};
    int mirror_parity = 0;
    uint16_t *d_consumer_lut = nullptr;
    int32_t *d_consumer_slot = nullptr;  // the ring position the render kernels write (base.consumer_slot_dev)
    int64_t consumer_steps = 0;          // host count of the steps issued since the consumer output was set
    int32_t consumer_slot = 0;           // consumer_steps mod k: the device slot while every step is issued eagerly
    bool have_host_bufs = false;
    bool rgb_copy_enqueued = false;  // this step's observation DMA already follows the render kernels
    bool ob_direct = false;      // caller's obs block is contiguous and page-locked: DMA straight into it
    bool ob_registered = false;
    std::vector<void *> h_ob, h_ac;
    std::vector<std::vector<void *>> h_info;  // [space][env]
    float *h_rew = nullptr;
    uint8_t *h_first = nullptr;
    // pinned staging
    uint8_t *st_rgb = nullptr;
    int32_t *st_action = nullptr;
    float *st_rew = nullptr;
    uint8_t *st_first = nullptr;
    int32_t *st_prev_seed = nullptr;
    uint8_t *st_prev_complete = nullptr;
    int32_t *st_seed = nullptr;
    // state transfers (get_state / set_state and their batched forms): device and pinned staging of state_stage_bytes
    // each, grown by a transfer that needs more up to a fixed budget, and the blobs pgb200_get_states hands out
    unsigned char *d_state_stage = nullptr, *h_state_stage = nullptr;
    size_t state_stage_bytes = 0;
    std::vector<char> state_blobs;
    std::vector<int64_t> state_offsets;
    // snapshot slots: allocated by the first pgb200_get_snapshots (snaps.slots null until then), snap_bytes in all
    SnapshotStore snaps{};
    int64_t snap_bytes = 0;

    VecEnv() = default;
    VecEnv(const VecEnv &) = delete;
    VecEnv &operator=(const VecEnv &) = delete;
    ~VecEnv() {
        for (void *ptr : owned_dev) dev_free(ptr);
        for (void *ptr : owned_pinned) pinned_free(ptr);
        for (Event e : owned_events) event_destroy(e);
        for (Stream s : owned_streams) stream_destroy(s);
    }

    // A device array of n elements (at least one), zero-filled on the legacy stream, that the handle owns
    template <class T>
    T *alloc(size_t n) {
        const size_t bytes = (n ? n : 1) * sizeof(T);
        void *ptr = dev_malloc(bytes);
        owned_dev.push_back(ptr);
        dev_memset(ptr, 0, bytes);
        return (T *)ptr;
    }
    // A pinned host buffer of n elements (at least one) that the handle owns
    template <class T>
    T *alloc_pinned(size_t n) {
        void *ptr = pinned_alloc((n ? n : 1) * sizeof(T));
        owned_pinned.push_back(ptr);
        return (T *)ptr;
    }
    Stream own(Stream s) {
        owned_streams.push_back(s);
        return s;
    }
    Event own(Event e) {
        owned_events.push_back(e);
        return e;
    }

    LaunchCtx lctx() {
        LaunchCtx lc;
        lc.stream = stream;
        lc.logic_stream = nullptr;
        lc.link = nullptr;
        lc.max_logic_blocks = max_logic_blocks;
        lc.num_sms = num_sms;
        lc.render_smem_floor = render_smem_floor;
        lc.tev = nullptr;
        lc.ticket = d_tickets;
        lc.launch_counter = &launches;
        lc.look_stream = nullptr;
        lc.look_fork = nullptr;
        return lc;
    }

    // `base` as the launches of joint game g see it: the game's assets, id and fixed asset seed, and its slots of the
    // level bank and of level lookahead where they exist. The caller sets the launch's env range (and, for lookahead,
    // the launch's segment of the list and its staging).
    KParams game_params(int g) const {
        KParams p = base;
        p.assets = d_assets[g];
        p.game_id = games[g]->id;
        p.fixed_asset_seed = fnv1a(games[g]->name);
        if (base.bank.slots)
            p.bank = banks[g];
        if (base.look.slot.slots)
            p.look.slot = looks[g].slot;
        return p;
    }

    // The kernels the next step runs: the opt-ins `base` holds. This is the one place that reads their pointers as
    // switches, and each entry point that turns one on assigns the pointer read here last, once the feature's arrays
    // are complete, so that no step sees a half-built feature.
    StepShape step_shape(bool init) const {
        StepShape s;
        s.init = init;
        if (init)
            return s;
        s.level_choice = base.next_level_seed != nullptr;
        s.pause = base.pause != nullptr;
        s.final_outputs = base.level_end != nullptr;
        s.bank = base.bank.slots != nullptr;
        s.look = base.look.slot.slots != nullptr;
        s.roll = base.roll.rgb != nullptr;
        s.repeat = base.repeat != nullptr;
        return s;
    }

    // One step = for every (game, env chunk): logic kernel then render kernel. Chunks go round-robin
    // onto a few auxiliary streams forked from / joined to the handle's stream with events, so the
    // latency-bound logic kernel of one chunk overlaps the issue-bound render kernel of another on
    // the same SMs (the two kernels stress different limits; back to back they leave both idle).
    void launch(bool init) {
        const int G = (int)games.size();
        const int per_game = num_envs / G;
        int chunks = force_chunks > 0 ? force_chunks : kChunks;
        if (force_chunks <= 0 && per_game < 4096 * chunks)
            chunks = 1;
        // more than one (logic, render) pair in the step — env chunks of one game, or the games of a
        // joint list — are spread over the auxiliary streams so they overlap on the SMs
        const int nstreams = (chunks * G > 1 && !serialize_launches) ? kAuxStreams : 0;
        const StepShape shape = step_shape(init);
#ifndef PG_HOSTSIM
        // the consumer ring moves on once per step, behind the previous step and ahead of every render
        // kernel of this one (they all start after the fork below)
        if (!init && base.consumer) {
            ring_advance_kernel<<<1, 1, 0, stream>>>(d_consumer_slot, base.consumer_k);
            CUDA_CHECK(cudaGetLastError());
            launches++;
        }
        // so does the rollout's cursor
        if (shape.roll) {
            ring_advance_kernel<<<1, 1, 0, stream>>>(base.roll.cursor, base.roll.slots);
            CUDA_CHECK(cudaGetLastError());
            launches++;
        }
        if (nstreams) {
            CUDA_CHECK(cudaEventRecord(ev_fork, stream));
            for (int s = 0; s < nstreams; s++) {
                CUDA_CHECK(cudaStreamWaitEvent(aux[s], ev_fork, 0));
                if (priority_split)
                    CUDA_CHECK(cudaStreamWaitEvent(aux_hi[s], ev_fork, 0));
            }
        }
#else
        if (shape.roll) {
            *base.roll.cursor = (*base.roll.cursor + 1) % base.roll.slots;
            launches++;
        }
#endif
        if (!init && mirror[0])
            mirror_parity ^= 1;
        if (!init && base.consumer) {
            consumer_steps++;
            consumer_slot = (int32_t)(consumer_steps % base.consumer_k);
        }
        int k = 0;
        for (int g = 0; g < G; g++) {
            for (int cidx = 0; cidx < chunks; cidx++, k++) {
                const int lo = (int)((int64_t)per_game * cidx / chunks);
                const int hi = (int)((int64_t)per_game * (cidx + 1) / chunks);
                KParams p = game_params(g);
                p.env_first = g + lo * G;
                p.env_step = G;
                p.env_count = hi - lo;
                if (shape.two_phase())
                    p.reset_list = base.reset_list + g * per_game + lo;  // the launch's own segment
                LaunchCtx lc = lctx();
                lc.ticket = d_tickets + k % kMaxTickets;
                if (shape.look) {
                    // launches that share a side stream run their lookahead kernels one after the other
                    const int side = k % kAuxStreams;
                    p.look.list = base.look.list + g * per_game + lo;
                    p.look.stage = base.look.stage + side * look_stage_bytes;
                    lc.look_stream = look_side[side];
                    lc.look_fork = look_fork[side];
                }
                if (nstreams) {
                    lc.stream = aux[k % nstreams];
                    if (priority_split) {
                        lc.logic_stream = aux_hi[k % nstreams];
                        lc.link = ev_link[k % nstreams];
                    }
                }
                if (timing && !shape.final_outputs && tev_used + 4 <= tev_pool.size()) {
                    lc.tev = &tev_pool[tev_used];
                    tev_used += 4;
                    tev_envs.push_back(p.env_count);
                }
                games[g]->step[view[g]](p, lc, shape);
#ifndef PG_HOSTSIM
                // libenv (host buffer) mode: start this chunk's observation DMA right behind its
                // render kernel, on the same stream, so the copy of one chunk overlaps the kernels
                // of the next instead of waiting for the whole step (PCIe is the e2e bottleneck:
                // 12 KiB per env and step)
                if (!init && mirror[0] && hi > lo) {
                    // the gather of SURVEY §8e without a collective: this launch's frames go straight
                    // to their place in the destination rank's buffer, overlapping the other launches
                    const size_t frame = RES_W * RES_H * 3;
                    const size_t first = (size_t)(g + lo * G) * frame;
                    if (G == 1)
                        CUDA_CHECK(cudaMemcpyAsync(mirror[mirror_parity] + first, base.rgb + first, (size_t)(hi - lo) * frame,
                                                   cudaMemcpyDeviceToDevice, lc.stream));
                    else
                        CUDA_CHECK(cudaMemcpy2DAsync(mirror[mirror_parity] + first, (size_t)G * frame, base.rgb + first, (size_t)G * frame, frame,
                                                     (size_t)(hi - lo), cudaMemcpyDeviceToDevice, lc.stream));
                }
                if (have_host_bufs && G == 1 && hi > lo) {
                    const size_t frame = RES_W * RES_H * 3;
                    uint8_t *rgb_dst = ob_direct ? (uint8_t *)h_ob[0] : st_rgb;
                    CUDA_CHECK(cudaMemcpyAsync(rgb_dst + (size_t)lo * frame, base.rgb + (size_t)lo * frame, (size_t)(hi - lo) * frame,
                                               cudaMemcpyDeviceToHost, lc.stream));
                    rgb_copy_enqueued = true;
                }
                // the lookahead kernel joins the launch's stream behind everything above, which never waits for it;
                // the step still ends with it, so that a captured step is self-contained
                if (shape.look && hi > lo) {
                    CUDA_CHECK(cudaEventRecord(look_join[k % kAuxStreams], lc.look_stream));
                    CUDA_CHECK(cudaStreamWaitEvent(lc.stream, look_join[k % kAuxStreams], 0));
                }
#endif
            }
        }
#ifndef PG_HOSTSIM
        if (nstreams) {
            for (int s = 0; s < nstreams; s++) {
                CUDA_CHECK(cudaEventRecord(ev_join[s], aux[s]));
                CUDA_CHECK(cudaStreamWaitEvent(stream, ev_join[s], 0));
            }
        }
#endif
    }

    void ensure_initial_reset() {
        if (initial_reset_done)
            return;
        launch(true);
        initial_reset_done = true;
    }

    void sync() { stream_sync(stream); }

    // True while the handle's stream captures a CUDA graph. The entry points that wait for the device or
    // allocate then refuse (-1, or a fatal message where the call returns nothing): either would
    // invalidate the caller's capture.
    bool capturing() { return stream_capturing(stream); }
    void refuse_in_capture(const char *what) {
        if (capturing())
            pg_fatal("%s cannot run while the handle's stream is capturing a CUDA graph\n", what);
    }

    // The start of an entry point that waits for the device and returns an error value (-1, or UINT32_MAX): false
    // while the handle's stream captures. Otherwise true once the stream has finished its work, the initial reset
    // included when `initial_reset` asks for it.
    bool try_sync(bool initial_reset = false) {
        if (capturing())
            return false;
        if (initial_reset)
            ensure_initial_reset();
        sync();
        return true;
    }

    // The start of an entry point that hands out an opt-in array: false (the entry point returns -1) while the
    // handle's stream captures, unless the array is already allocated (`allocated`) and the initial reset has run,
    // since either would invalidate the caller's capture. Then the initial reset.
    bool begin_opt_in(bool allocated) {
        if ((!initial_reset_done || !allocated) && capturing())
            return false;
        ensure_initial_reset();
        return true;
    }

    // An opt-in per-env array of `per_env` elements per env that the handle owns, allocated at the first request
    // (ptr null) with every byte set to `fill` on the handle's stream, which completes before the caller uses it
    // from any stream
    template <class T>
    void opt_in_array(T *&ptr, size_t per_env, int fill) {
        if (ptr)
            return;
        const size_t bytes = (num_envs ? (size_t)num_envs : 1) * per_env * sizeof(T);
        ptr = (T *)dev_malloc(bytes);
        owned_dev.push_back(ptr);
        memset_async(ptr, fill, bytes, stream);
        sync();
    }

    // The state transfers' staging, at least `bytes` of each kind; a smaller one is released first. Called with the
    // handle's stream idle.
    void grow_state_stage(size_t bytes) {
        if (bytes <= state_stage_bytes)
            return;
        auto drop = [](std::vector<void *> &owned, void *ptr) { owned.erase(std::find(owned.begin(), owned.end(), ptr)); };
        if (d_state_stage) {
            drop(owned_dev, d_state_stage);
            dev_free(d_state_stage);
            drop(owned_pinned, h_state_stage);
            pinned_free(h_state_stage);
        }
        d_state_stage = (unsigned char *)dev_malloc(bytes);
        owned_dev.push_back(d_state_stage);
        h_state_stage = alloc_pinned<unsigned char>(bytes);
        state_stage_bytes = bytes;
    }

    void set_device() { set_current_device(device); }
};

std::string default_pack_path() {
    // <dir of this .so>/data/assets.pack, overridable with PROCGEN_B200_ASSET_PACK
    const char *e = getenv("PROCGEN_B200_ASSET_PACK");
    if (e && e[0])
        return e;
    Dl_info info;
    if (dladdr((void *)&libenv_version, &info) && info.dli_fname) {
        std::string so(info.dli_fname);
        size_t slash = so.rfind('/');
        std::string dir = slash == std::string::npos ? "." : so.substr(0, slash);
        return dir + "/data/assets.pack";
    }
    return "assets.pack";
}

void fill_tensortypes(VecEnv *v) {
    // vecgame.cpp:212-268
    libenv_tensortype s;
    memset(&s, 0, sizeof(s));
    strcpy(s.name, "rgb");
    s.scalar_type = LIBENV_SCALAR_TYPE_DISCRETE;
    s.dtype = LIBENV_DTYPE_UINT8;
    s.shape[0] = RES_W;
    s.shape[1] = RES_H;
    s.shape[2] = 3;
    s.ndim = 3;
    s.low.uint8 = 0;
    s.high.uint8 = 255;
    v->observation_types.push_back(s);

    memset(&s, 0, sizeof(s));
    strcpy(s.name, "action");
    s.scalar_type = LIBENV_SCALAR_TYPE_DISCRETE;
    s.dtype = LIBENV_DTYPE_INT32;
    s.ndim = 0;
    s.low.int32 = 0;
    s.high.int32 = v->num_actions - 1;
    v->action_types.push_back(s);

    const char *info_names[3] = {"prev_level_seed", "prev_level_complete", "level_seed"};
    for (int i = 0; i < 3; i++) {
        memset(&s, 0, sizeof(s));
        strcpy(s.name, info_names[i]);
        s.scalar_type = LIBENV_SCALAR_TYPE_DISCRETE;
        s.ndim = 0;
        if (i == 1) {
            s.dtype = LIBENV_DTYPE_UINT8;
            s.low.uint8 = 0;
            s.high.uint8 = 1;
        } else {
            s.dtype = LIBENV_DTYPE_INT32;
            s.low.int32 = 0;
            s.high.int32 = INT32_MAX;
        }
        v->info_types.push_back(s);
    }
}

}  // namespace

// ================================================================= C ABI
extern "C" {

int libenv_version(void) { return LIBENV_VERSION; }

int pgb200_is_device_build(void) { return kDeviceBuild; }

libenv_env *libenv_make(int num_envs, const struct libenv_options options) {
    OptParser opts(options);
    VecEnv *v = new VecEnv;
    v->num_envs = num_envs;

    // ---- VecGame::VecGame options (vecgame.cpp:169-190)
    std::string env_name, resource_root;
    int32_t num_levels = 0, start_level = -1, rand_seed = 0, num_threads = 4;
    bool render_human = false;
    opts.consume_string("env_name", &env_name);
    opts.consume_int("num_levels", &num_levels);
    opts.consume_int("start_level", &start_level);
    opts.consume_int("num_actions", &v->num_actions);
    opts.consume_int("rand_seed", &rand_seed);
    opts.consume_int("num_threads", &num_threads);
    opts.consume_string("resource_root", &resource_root);
    opts.consume_bool("render_human", &render_human);
    // ---- backend extensions
    int32_t cuda_device = -1, env_index_offset = 0, env_index_total = -1;
    bool snap = true;
    opts.consume_int("cuda_device", &cuda_device);
    opts.consume_int("env_index_offset", &env_index_offset);
    opts.consume_int("env_index_total", &env_index_total);
    opts.consume_bool("snap_target_rect", &snap);
    if (env_index_total < 0)
        env_index_total = env_index_offset + num_envs;

    pg_fassert(num_threads >= 0);
    pg_fassert(env_name != "");
    pg_fassert(v->num_actions > 0);
    pg_fassert(num_levels >= 0);
    pg_fassert(start_level >= 0);
    if (render_human)
        pg_fatal("render_human (512x512 antialiased info['rgb']) is not supported by procgen_b200\n");

    // ---- Game::parse_options (game.cpp:42-75)
    bool use_easy_jump = false, paint_vel_info = false, use_generated_assets = false, use_monochrome_assets = false;
    bool restrict_themes = false, use_backgrounds = true, center_agent = false, use_sequential_levels = false;
    opts.consume_bool("use_easy_jump", &use_easy_jump);
    opts.consume_bool("paint_vel_info", &paint_vel_info);
    opts.consume_bool("use_generated_assets", &use_generated_assets);
    opts.consume_bool("use_monochrome_assets", &use_monochrome_assets);
    opts.consume_bool("restrict_themes", &restrict_themes);
    opts.consume_bool("use_backgrounds", &use_backgrounds);
    opts.consume_bool("center_agent", &center_agent);
    opts.consume_bool("use_sequential_levels", &use_sequential_levels);
    int32_t dist_mode = EasyMode, plain_assets = 0, physics_mode = 0, debug_mode = 0, game_type = 0;
    opts.consume_int("distribution_mode", &dist_mode);
    opts.consume_int("plain_assets", &plain_assets);
    opts.consume_int("physics_mode", &physics_mode);
    opts.consume_int("debug_mode", &debug_mode);
    opts.consume_int("game_type", &game_type);
    opts.ensure_empty();
    if (use_generated_assets)
        pg_fatal("use_generated_assets is not supported by procgen_b200\n");

    std::vector<std::string> env_names = split(env_name, ",");
    const int G = (int)env_names.size();
    pg_fassert(num_envs % G == 0);
    pg_fassert(env_index_offset % G == 0);
    for (const auto &name : env_names) {
        const GameVTable *g = find_game(name);
        if (!g)
            pg_fatal("unknown or not yet supported env_name '%s'\n", name.c_str());
        // Five games honour center_agent=false by drawing their whole (up to 64x64-cell) world
        // (basic-abstract-game.cpp:819-838) through the render path sized for that view.
        int view = 0;
        if (!center_agent && (name == "coinrun" || name == "climber" || name == "caveflyer" || name == "jumper" || name == "ninja")) {
            if (g->step[1] == nullptr)
                pg_fatal("center_agent=false is not supported for '%s' by procgen_b200 yet\n", name.c_str());
            view = 1;
        }
        v->view.push_back(view);
        // mode validity, game.cpp:56-66
        if (dist_mode == EasyMode || dist_mode == HardMode) {
        } else if (dist_mode == ExtremeMode) {
            pg_fassert(name == "chaser" || name == "dodgeball" || name == "leaper" || name == "starpilot");
        } else if (dist_mode == MemoryMode) {
            pg_fassert(name == "caveflyer" || name == "dodgeball" || name == "heist" || name == "jumper" || name == "maze" || name == "miner");
        } else {
            pg_fatal("invalid distribution_mode %d\n", dist_mode);
        }
        v->games.push_back(g);
    }

    // ---- device
#ifndef PG_HOSTSIM
    if (cuda_device < 0)
        CUDA_CHECK(cudaGetDevice(&cuda_device));
    v->device = cuda_device;
    v->set_device();
    auto new_stream = [v] {
        cudaStream_t s = nullptr;
        CUDA_CHECK(cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking));
        return v->own(s);
    };
    auto new_event = [v] {
        cudaEvent_t e = nullptr;
        CUDA_CHECK(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
        return v->own(e);
    };
    v->stream = v->own_stream = new_stream();
    {
        const char *e = getenv("PGB200_PRIORITY_SPLIT");
        v->priority_split = e && atoi(e) != 0;
    }
    int prio_lo = 0, prio_hi = 0;
    CUDA_CHECK(cudaDeviceGetStreamPriorityRange(&prio_lo, &prio_hi));  // numerically lower = higher priority
    for (int s = 0; s < VecEnv::kAuxStreams; s++) {
        v->aux[s] = new_stream();
        v->ev_join[s] = new_event();
        if (v->priority_split) {
            cudaStream_t hi = nullptr;
            CUDA_CHECK(cudaStreamCreateWithPriority(&hi, cudaStreamNonBlocking, prio_hi));
            v->aux_hi[s] = v->own(hi);
            v->ev_link[s] = new_event();
        }
    }
    v->ev_fork = new_event();
    {
        cudaDeviceProp prop;
        CUDA_CHECK(cudaGetDeviceProperties(&prop, v->device));
        v->max_logic_blocks = prop.multiProcessorCount * PG_LOGIC_MIN_BLOCKS;
        v->num_sms = prop.multiProcessorCount;
        // tuning knobs (defaults chosen by sweeping them with bench.py): resident logic blocks and
        // render CTAs per SM
        if (const char *e = getenv("PGB200_LOGIC_BLOCKS_PER_SM"))
            if (atoi(e) > 0)
                v->max_logic_blocks = prop.multiProcessorCount * atoi(e);
        int render_ctas = PG_RENDER_CTAS_PER_SM;
        if (const char *e = getenv("PGB200_RENDER_CTAS_PER_SM"))
            render_ctas = atoi(e);
        if (render_ctas > 0 && render_ctas < 16) {
            // usable shared memory per SM is 227 KiB, each CTA also pays 1 KiB of system reserve
            v->render_smem_floor = (227 * 1024) / render_ctas - 1024 - 16;
            v->render_smem_floor &= ~15;
        }
        v->d_consumer_slot = v->alloc<int32_t>(1);
        v->base.consumer_slot_dev = v->d_consumer_slot;
    }
    // sub_step <-> push_obj recurse to depth 5 on the logic thread
    {
        size_t cur = 0;
        CUDA_CHECK(cudaDeviceGetLimit(&cur, cudaLimitStackSize));
        if (cur < 4096)  // only ever raise it: the host application may have asked for more
            CUDA_CHECK(cudaDeviceSetLimit(cudaLimitStackSize, 4096));
    }
#endif
    v->d_tickets = v->alloc<TicketSlot>(VecEnv::kMaxTickets);

    // ---- assets
    std::string pack_path = resource_root;
    if (pack_path.size() >= 5 && pack_path.compare(pack_path.size() - 5, 5, ".pack") == 0) {
    } else if (!pack_path.empty()) {
        if (pack_path.back() != '/')
            pack_path += "/";
        pack_path += "assets.pack";
    } else {
        pack_path = default_pack_path();
    }
    try {
        host::AssetPackReader pack(pack_path);
        host::AtlasBuilder atlas(pack);
        std::vector<GameAssets> tables(G);
        for (int g = 0; g < G; g++) atlas.build_game(v->games[g]->id, tables[g]);
        uint32_t *atlas_texels = v->alloc<uint32_t>(atlas.texels.size());
        copy_to_dev(atlas_texels, atlas.texels.data(), atlas.texels.size() * sizeof(uint32_t));
        v->base.atlas = atlas_texels;
        for (int g = 0; g < G; g++) {
            GameAssets *d = v->alloc<GameAssets>(1);
            copy_to_dev(d, &tables[g], sizeof(GameAssets));
            v->d_assets.push_back(d);
        }
        // pre-scaled cell tiles of every sprite (pg_raster.cuh TileTable), filled on the device by
        // the general blit path's own arithmetic
        const bool want_tiles = !(getenv("PGB200_NO_TILES") && atoi(getenv("PGB200_NO_TILES")) != 0);
        const int S = (int)atlas.tile_sprites.size();
        if (want_tiles && S > 0) {
            std::vector<uint32_t> index((size_t)S * TILE_VARIANTS);
            size_t top = 0;
            for (int sl = 0; sl < S; sl++)
                for (int tw = 1; tw <= MAX_TILE_DIM; tw++)
                    for (int th = 1; th <= MAX_TILE_DIM; th++) {
                        index[((size_t)sl * MAX_TILE_DIM + (tw - 1)) * MAX_TILE_DIM + (th - 1)] = (uint32_t)top;
                        top += (size_t)tile_words(tw, th);
                    }
            if (top >= (size_t)1 << 32)
                throw std::runtime_error("tile table too large");
            uint32_t *tile_index = v->alloc<uint32_t>(index.size());
            copy_to_dev(tile_index, index.data(), index.size() * sizeof(uint32_t));
            SpriteDesc *tile_sprites = v->alloc<SpriteDesc>((size_t)S);
            copy_to_dev(tile_sprites, atlas.tile_sprites.data(), (size_t)S * sizeof(SpriteDesc));
            uint32_t *tile_texels = v->alloc<uint32_t>(top);
#ifndef PG_HOSTSIM
            tile_table_kernel<<<S * TILE_VARIANTS, 64>>>(tile_sprites, tile_index, tile_texels, atlas_texels);
            CUDA_CHECK(cudaGetLastError());
#else
            for (int sl = 0; sl < S; sl++)
                for (int vv = 0; vv < TILE_VARIANTS; vv++)
                    tile_table_fill(tile_sprites, tile_index, tile_texels, atlas_texels, sl, vv / MAX_TILE_DIM + 1, vv % MAX_TILE_DIM + 1, 0, 1);
#endif
            v->base.tiles.texels = tile_texels;
            v->base.tiles.index = tile_index;
            v->base.tiles.sprites = tile_sprites;
            v->base.tiles.n_slots = S;
        }
    } catch (const std::exception &e) {
        pg_fatal("failed to load images %s\n", e.what());
    }

    fill_tensortypes(v);

    // ---- state arrays
    int ent_cap = 0, grid_cap = 0, scratch_words = 0, rot_records = 0, blit_records = 0, setup_bytes = 0, cell_records = 0;
    for (const auto &g : v->games) {
        rot_records = std::max(rot_records, g->rot_records);
        blit_records = std::max(blit_records, g->blit_records);
        const int vw = v->view[&g - &v->games[0]];
        setup_bytes = std::max(setup_bytes, g->setup_bytes[vw]);
        cell_records = std::max(cell_records, g->cell_records[vw]);
        ent_cap = std::max(ent_cap, g->ent_cap);
        grid_cap = std::max(grid_cap, g->grid_cap);
        scratch_words = std::max(scratch_words, g->scratch_words);
    }
    KParams &p = v->base;
    const size_t N = (size_t)num_envs;
    p.ent_stride = ent_cap + 1;
    p.grid_stride = grid_cap;
    p.scratch_stride = scratch_words;
    p.hdr = v->alloc<EnvHdr>(N);
    p.ents = v->alloc<Entity>(N * p.ent_stride);
    p.grid = v->alloc<int16_t>(N * p.grid_stride);
    p.rng = v->alloc<MT19937>(N);
    p.lvl_rng = v->alloc<MT19937>(N);
    p.scratch = v->alloc<int32_t>(N * (size_t)scratch_words);
    p.rot_stride = rot_records;
    p.rot_scratch = rot_records > 0 ? v->alloc<RotBlit>(N * (size_t)rot_records) : nullptr;
    p.blit_stride = blit_records;
    p.blit_list = v->alloc<Blit>(N * (size_t)blit_records);
    p.cell_spill_stride = cell_records;
    p.cell_spill = v->alloc<Blit>(N * (size_t)cell_records);
    p.frame_setup_stride = (setup_bytes + 15) & ~15;
    p.frame_setup = v->alloc<unsigned char>(N * (size_t)p.frame_setup_stride);
    v->d_action = v->alloc<int32_t>(N);
    p.action = v->d_action;
    p.rgb = v->alloc<uint8_t>(N * RES_W * RES_H * 3);
    p.rew = v->alloc<float>(N);
    p.first = v->alloc<uint8_t>(N);
    p.info_prev_level_seed = v->alloc<int32_t>(N);
    p.info_prev_level_complete = v->alloc<uint8_t>(N);
    p.info_level_seed = v->alloc<int32_t>(N);
    p.dbg_cycles = getenv("PGB200_DEBUG_TIMING") ? v->alloc<uint32_t>(N) : nullptr;

    // ---- per-env seed chain (vecgame.cpp:301-314), replayed for the global env indices
    {
        std::mt19937 game_level_seed_gen;
        game_level_seed_gen.seed((uint32_t)rand_seed);
        for (int i = 0; i < env_index_offset; i++) (void)game_level_seed_gen();
        std::vector<uint32_t> seeds(N);
        for (size_t i = 0; i < N; i++) seeds[i] = (uint32_t)game_level_seed_gen();
        uint32_t *lvl_seeds = v->alloc<uint32_t>(N);
        copy_to_dev(lvl_seeds, seeds.data(), N * sizeof(uint32_t));
        p.lvl_seeds = lvl_seeds;
    }

    // vecgame.cpp:284-293
    if (num_levels == 0) {
        p.level_seed_low = 0;
        p.level_seed_high = INT32_MAX;
    } else {
        p.level_seed_low = start_level;
        p.level_seed_high = start_level + num_levels;
    }
    memset(&p.options, 0, sizeof(p.options));
    p.options.paint_vel_info = paint_vel_info;
    p.options.use_generated_assets = use_generated_assets;
    p.options.use_monochrome_assets = use_monochrome_assets;
    p.options.restrict_themes = restrict_themes;
    p.options.use_backgrounds = use_backgrounds;
    p.options.center_agent = center_agent;
    p.options.use_sequential_levels = use_sequential_levels;
    p.options.debug_mode = debug_mode;
    v->const_fields.use_easy_jump = use_easy_jump;
    v->const_fields.plain_assets = plain_assets;
    v->const_fields.physics_mode = physics_mode;
    v->const_fields.game_type = game_type;
    p.options.distribution_mode = dist_mode;
    p.snap = snap ? 1 : 0;
    p.env_global_offset = env_index_offset;
    // every upload and memset above ran on the legacy default stream; the step kernels run on
    // non-blocking streams that do not order against it
    device_sync();
    return (libenv_env *)v;
}

int libenv_get_tensortypes(libenv_env *handle, enum libenv_space_name name, struct libenv_tensortype *out_types) {
    VecEnv *v = (VecEnv *)handle;
    const std::vector<libenv_tensortype> *types = nullptr;
    if (name == LIBENV_SPACE_OBSERVATION)
        types = &v->observation_types;
    else if (name == LIBENV_SPACE_ACTION)
        types = &v->action_types;
    else if (name == LIBENV_SPACE_INFO)
        types = &v->info_types;
    else
        return 0;
    if (out_types)
        for (size_t i = 0; i < types->size(); i++) out_types[i] = (*types)[i];
    return (int)types->size();
}

static void fetch_to_host(VecEnv *v) {
    const size_t N = (size_t)v->num_envs;
    const KParams &p = v->base;
    const size_t frame = RES_W * RES_H * 3;
    uint8_t *rgb_dst = v->ob_direct ? (uint8_t *)v->h_ob[0] : v->st_rgb;
    if (!v->rgb_copy_enqueued)
        copy_from_dev_async(rgb_dst, p.rgb, N * frame, v->stream);
    v->rgb_copy_enqueued = false;
    copy_from_dev_async(v->st_rew, p.rew, N * sizeof(float), v->stream);
    copy_from_dev_async(v->st_first, p.first, N, v->stream);
    copy_from_dev_async(v->st_prev_seed, p.info_prev_level_seed, N * 4, v->stream);
    copy_from_dev_async(v->st_prev_complete, p.info_prev_level_complete, N, v->stream);
    copy_from_dev_async(v->st_seed, p.info_level_seed, N * 4, v->stream);
    v->sync();
    if (!v->ob_direct)
        for (size_t e = 0; e < N; e++) memcpy(v->h_ob[e], v->st_rgb + e * frame, frame);
    memcpy(v->h_rew, v->st_rew, N * sizeof(float));
    memcpy(v->h_first, v->st_first, N);
    for (size_t e = 0; e < N; e++) {
        *(int32_t *)v->h_info[0][e] = v->st_prev_seed[e];
        *(uint8_t *)v->h_info[1][e] = v->st_prev_complete[e];
        *(int32_t *)v->h_info[2][e] = v->st_seed[e];
    }
}

void libenv_set_buffers(libenv_env *handle, struct libenv_buffers *bufs) {
    VecEnv *v = (VecEnv *)handle;
    v->set_device();
    v->refuse_in_capture("libenv_set_buffers");
    const size_t N = (size_t)v->num_envs;
    pg_fassert(!v->initial_reset_done);
    v->h_ob.assign(bufs->ob, bufs->ob + N);  // one observation space
    v->h_ac.assign(bufs->ac, bufs->ac + N);  // one action space
    v->h_info.resize(v->info_types.size());
    for (size_t s = 0; s < v->info_types.size(); s++) v->h_info[s].assign(bufs->info + s * N, bufs->info + (s + 1) * N);
    v->h_rew = bufs->rew;
    v->h_first = bufs->first;
    v->have_host_bufs = true;
    {
        // gym3 hands out one contiguous [N][64][64][3] array: page-lock it once and DMA into it
        // directly instead of bouncing 12 KiB/env through a staging buffer every step
        const size_t frame = RES_W * RES_H * 3;
        bool contiguous = true;
        for (size_t e = 1; e < N && contiguous; e++)
            contiguous = ((uint8_t *)v->h_ob[e] == (uint8_t *)v->h_ob[0] + e * frame);
        v->ob_direct = false;
#ifndef PG_HOSTSIM
        if (contiguous) {
            cudaPointerAttributes attr;
            if (cudaPointerGetAttributes(&attr, v->h_ob[0]) == cudaSuccess && attr.type == cudaMemoryTypeHost) {
                v->ob_direct = true;
            } else {
                cudaGetLastError();
                if (cudaHostRegister(v->h_ob[0], N * frame, cudaHostRegisterDefault) == cudaSuccess) {
                    v->ob_direct = true;
                    v->ob_registered = true;
                } else {
                    cudaGetLastError();
                }
            }
        }
#else
        v->ob_direct = contiguous;
#endif
    }
    v->st_rgb = v->ob_direct ? nullptr : v->alloc_pinned<uint8_t>(N * RES_W * RES_H * 3);
    v->st_action = v->alloc_pinned<int32_t>(N);
    v->st_rew = v->alloc_pinned<float>(N);
    v->st_first = v->alloc_pinned<uint8_t>(N);
    v->st_prev_seed = v->alloc_pinned<int32_t>(N);
    v->st_prev_complete = v->alloc_pinned<uint8_t>(N);
    v->st_seed = v->alloc_pinned<int32_t>(N);
    v->ensure_initial_reset();  // vecgame.cpp:349-353
}

void libenv_observe(libenv_env *handle) {
    VecEnv *v = (VecEnv *)handle;
    v->set_device();
    v->refuse_in_capture("libenv_observe");
    pg_fassert(v->have_host_bufs);
    fetch_to_host(v);
}

void libenv_act(libenv_env *handle) {
    VecEnv *v = (VecEnv *)handle;
    v->set_device();
    v->refuse_in_capture("libenv_act");
    pg_fassert(v->have_host_bufs);
    const size_t N = (size_t)v->num_envs;
    v->sync();  // staging buffer reuse (wait_for_stepping_threads, vecgame.cpp:379)
    for (size_t e = 0; e < N; e++) v->st_action[e] = *(int32_t *)v->h_ac[e];
    copy_to_dev_async(v->d_action, v->st_action, N * 4, v->stream);
    v->launch(false);
}

void libenv_close(libenv_env *handle) {
    VecEnv *v = (VecEnv *)handle;
    if (!v)
        return;
    v->set_device();
    v->refuse_in_capture("libenv_close");
    v->sync();
    if (v->ob_registered)
        host_unregister(v->h_ob[0]);
    delete v;  // releases everything the handle allocated or created
}

int pgb200_get_device_buffers(libenv_env *handle, struct pgb200_device_buffers *out) {
    VecEnv *v = (VecEnv *)handle;
    v->set_device();
    if (!v->initial_reset_done && v->capturing())
        return -1;
    v->ensure_initial_reset();
    const KParams &p = v->base;
    out->rgb = p.rgb;
    out->rew = p.rew;
    out->first = p.first;
    out->prev_level_seed = p.info_prev_level_seed;
    out->prev_level_complete = p.info_prev_level_complete;
    out->level_seed = p.info_level_seed;
    out->action = v->d_action;
    out->num_envs = v->num_envs;
    out->device = v->device;
    out->stream = (void *)v->stream;
    return 0;
}

int pgb200_get_next_level_seeds(libenv_env *handle, int32_t **out) {
    VecEnv *v = (VecEnv *)handle;
    v->set_device();
    if (!v->begin_opt_in(v->base.next_level_seed != nullptr))
        return -1;
    v->opt_in_array(v->base.next_level_seed, 1, 0xff);  // every entry -1
    *out = v->base.next_level_seed;
    return 0;
}

int pgb200_get_final_outputs(libenv_env *handle, struct pgb200_final_outputs *out) {
    VecEnv *v = (VecEnv *)handle;
    v->set_device();
    if (!v->begin_opt_in(v->base.level_end != nullptr))
        return -1;
    v->opt_in_array(v->base.final_rgb, RES_W * RES_H * 3, 0);
    v->opt_in_array(v->base.reset_list, 1, 0);
    v->opt_in_array(v->base.level_end, 1, 0);  // last: VecEnv::step_shape reads a non-null level_end as final outputs on
    out->rgb = v->base.final_rgb;
    out->level_end = v->base.level_end;
    return 0;
}

int pgb200_get_pause_mask(libenv_env *handle, uint8_t **out) {
    VecEnv *v = (VecEnv *)handle;
    v->set_device();
    if (!v->begin_opt_in(v->d_pause != nullptr))
        return -1;
    v->opt_in_array(v->base.paused, 1, 0);
    v->opt_in_array(v->d_pause, 1, 0);
    v->base.pause = v->d_pause;  // last: VecEnv::step_shape reads a non-null pause as the mask on
    *out = v->d_pause;
    return 0;
}

int pgb200_get_action_repeat(libenv_env *handle, int32_t **out) {
    VecEnv *v = (VecEnv *)handle;
    v->set_device();
    if (!v->begin_opt_in(v->d_repeat != nullptr))
        return -1;
    if (!v->d_repeat) {
        v->opt_in_array(v->d_repeat, 1, 0);
        const std::vector<int32_t> ones((size_t)std::max(v->num_envs, 1), 1);
        copy_to_dev_async(v->d_repeat, ones.data(), ones.size() * sizeof(int32_t), v->stream);
        v->sync();
    }
    v->base.repeat = v->d_repeat;  // last: VecEnv::step_shape reads a non-null repeat as action repeat on
    *out = v->d_repeat;
    return 0;
}

int pgb200_get_rollout(libenv_env *handle, int slots, struct pgb200_rollout *out) {
    VecEnv *v = (VecEnv *)handle;
    v->set_device();
    Rollout &r = v->base.roll;
    const size_t frame = RES_W * RES_H * 3, N = (size_t)std::max(v->num_envs, 1);
    if (slots < 2 || (r.rgb && slots != r.slots) || (size_t)slots > SIZE_MAX / (N * frame))
        return -1;
    if (!v->begin_opt_in(r.rgb != nullptr))
        return -1;
    if (!r.rgb) {
        uint8_t *rgb = nullptr;
        v->opt_in_array(rgb, (size_t)slots * frame, 0);
        v->opt_in_array(r.rew, (size_t)slots, 0);
        v->opt_in_array(r.first, (size_t)slots, 0);
        r.cursor = v->alloc<int32_t>(1);  // slot 0
        device_sync();                     // alloc's memset ran on the legacy stream
        r.slots = slots;
        r.num_envs = v->num_envs;
        // slot 0 holds the outputs current now: those of the last step issued, or of the initial reset
        copy_dev_async(rgb, v->base.rgb, (size_t)v->num_envs * frame, v->stream);
        copy_dev_async(r.rew, v->base.rew, (size_t)v->num_envs * sizeof(float), v->stream);
        copy_dev_async(r.first, v->base.first, (size_t)v->num_envs, v->stream);
        v->sync();
        r.rgb = rgb;  // last: VecEnv::step_shape reads a non-null rgb as the rollout on
    }
    out->rgb = r.rgb;
    out->rew = r.rew;
    out->first = r.first;
    out->cursor = r.cursor;
    return 0;
}

int pgb200_build_level_bank(libenv_env *handle, const int32_t *seeds, int count, int capacity) {
    VecEnv *v = (VecEnv *)handle;
    v->set_device();
    if (count < 0 || capacity < 0 || (count > 0 && !seeds))
        return -1;
    for (int i = 0; i < count; i++)
        if (seeds[i] < 0)
            return -1;
    std::vector<int32_t> sorted(seeds, seeds + count);
    std::sort(sorted.begin(), sorted.end());
    sorted.erase(std::unique(sorted.begin(), sorted.end()), sorted.end());
    const int n = (int)sorted.size();
    if (v->base.bank.slots ? n > v->bank_capacity : std::max(count, capacity) == 0)
        return -1;  // more distinct seeds than the capacity, or a first call that would fix it at 0
    if (!v->begin_opt_in(false))  // a build waits for the device, so it never runs under capture
        return -1;
    KParams &base = v->base;
    const int G = (int)v->games.size();
    if (!base.bank.slots) {
        v->bank_capacity = std::max(count, capacity);
        v->d_bank_seeds = v->alloc<int32_t>((size_t)v->bank_capacity);
        v->d_bank_count = v->alloc<int32_t>(1);
        // a banked step lists its resets as a step with final outputs does (launch_step)
        v->opt_in_array(base.bank_level_end, 1, 0);
        v->opt_in_array(base.reset_list, 1, 0);
        size_t total = 0;
        for (const GameVTable *g : v->games) {
            LevelBank b = slot_layout(g, base.options);
            b.seeds = v->d_bank_seeds;
            b.count = v->d_bank_count;
            b.slots = reinterpret_cast<unsigned char *>(total);  // offset until the allocation below
            total += (size_t)v->bank_capacity * b.slot_bytes;
            v->banks.push_back(b);
        }
        unsigned char *slots = v->alloc<unsigned char>(total);
        for (LevelBank &b : v->banks) b.slots = slots + reinterpret_cast<size_t>(b.slots);
        v->bank_bytes = (int64_t)total + (int64_t)v->bank_capacity * (int64_t)sizeof(int32_t) + (int64_t)sizeof(int32_t);
        // set last: VecEnv::step_shape reads a non-null slots pointer as the bank on
        base.bank = v->banks[0];
        base.bank.slots = slots;
        device_sync();  // alloc's memsets ran on the legacy stream
    }
    // staging of the build's warps (a level generated at the env's own capacities), bounded by a fixed budget, and
    // released when the build has finished with it
    const size_t stage_bytes = bank_stage_bytes(base);
    int warps = (int)std::min<size_t>((size_t)std::max(n, 1), std::max<size_t>(((size_t)256 << 20) / stage_bytes, 1));
    warps = std::min(warps, v->max_logic_blocks * kLogicEnvsPerBlock);
    std::unique_ptr<unsigned char, void (*)(void *)> stage((unsigned char *)dev_malloc((size_t)warps * stage_bytes), dev_free);
    // ordered behind every step issued so far, and every later step behind the rebuild
    copy_to_dev_async(v->d_bank_seeds, sorted.data(), (size_t)n * sizeof(int32_t), v->stream);
    for (int g = 0; g < G; g++) {
        LaunchCtx lc = v->lctx();
        v->games[g]->bank_build(v->game_params(g), lc, stage.get(), warps, n);
    }
    const int32_t n_dev = n;
    copy_to_dev_async(v->d_bank_count, &n_dev, sizeof(int32_t), v->stream);
    v->sync();  // the host sources above, then the staging
    v->bank_levels = n;
    return 0;
}

int pgb200_enable_level_lookahead(libenv_env *handle) {
    VecEnv *v = (VecEnv *)handle;
    v->set_device();
    KParams &base = v->base;
    if (base.look.slot.slots)
        return 0;
    if (!v->begin_opt_in(false))  // the fill waits for the device, so it never runs under capture
        return -1;
    const int G = (int)v->games.size();
    const int per_game = v->num_envs / G;
    // a lookahead handle lists its resets as a banked one does (launch_step)
    v->opt_in_array(base.bank_level_end, 1, 0);
    v->opt_in_array(base.reset_list, 1, 0);
    v->opt_in_array(base.look.list, 1, 0);
    size_t total = 0;
    for (const GameVTable *g : v->games) {
        LevelLookahead l{};
        l.slot = slot_layout(g, base.options);
        l.slot.slots = reinterpret_cast<unsigned char *>(total);  // offset until the allocation below
        total += (size_t)per_game * l.slot.slot_bytes;
        v->looks.push_back(l);
    }
    unsigned char *slots = v->alloc<unsigned char>(total);
    for (LevelLookahead &l : v->looks) {
        l.slot.slots = slots + reinterpret_cast<size_t>(l.slot.slots);
        memset_strided(l.slot.slots + sizeof(int32_t), 0xff, sizeof(int32_t), (size_t)l.slot.slot_bytes, (size_t)per_game);  // keys -1
    }
    // per-step staging: as many warps per side stream as a quarter of the bank build's budget allows, at most what
    // a launch's resets need at once
    const size_t stage_bytes = bank_stage_bytes(base);
    v->look_warps = (int)std::min<size_t>(std::max<size_t>(((size_t)64 << 20) / ((size_t)VecEnv::kAuxStreams * stage_bytes), 1), 128);
    v->look_warps = std::min(v->look_warps, v->max_logic_blocks * kLogicEnvsPerBlock);
    v->look_stage_bytes = (size_t)v->look_warps * stage_bytes;
    unsigned char *step_stage = v->alloc<unsigned char>(VecEnv::kAuxStreams * v->look_stage_bytes);
    v->d_look_served = v->alloc<unsigned long long>(3);
    v->look_bytes = (int64_t)total + (int64_t)(VecEnv::kAuxStreams * v->look_stage_bytes) + (int64_t)v->num_envs * (int64_t)sizeof(int32_t) +
                    3 * (int64_t)sizeof(unsigned long long);
#ifndef PG_HOSTSIM
    // The side streams the lookahead kernels run on beside the frames. Render CTAs fill the SMs, and a stream's
    // priority decides whose pending blocks are placed first: at high priority the generation warps start as soon as
    // a slot frees, and the step (which ends with them) is faster than at low priority (DESIGN §7).
    int prio_lo = 0, prio_hi = 0;
    CUDA_CHECK(cudaDeviceGetStreamPriorityRange(&prio_lo, &prio_hi));
    const int prio = prio_hi;
    for (int s = 0; s < VecEnv::kAuxStreams; s++) {
        cudaStream_t st = nullptr;
        CUDA_CHECK(cudaStreamCreateWithPriority(&st, cudaStreamNonBlocking, prio));
        v->look_side[s] = v->own(st);
        cudaEvent_t e[2];
        for (cudaEvent_t &ev : e) {
            CUDA_CHECK(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
            v->own(ev);
        }
        v->look_fork[s] = e[0];
        v->look_join[s] = e[1];
    }
#endif
    device_sync();  // alloc's memsets ran on the legacy stream
    base.look.games = G;
    base.look.stage = step_stage;
    base.look.stage_warps = v->look_warps;
    base.look.served = v->d_look_served;
    // the bulk fill: every env's next level predicted, then generated with the bank build's staging budget
    int warps = (int)std::min<size_t>((size_t)std::max(per_game, 1), std::max<size_t>(((size_t)256 << 20) / stage_bytes, 1));
    warps = std::min(warps, v->max_logic_blocks * kLogicEnvsPerBlock);
    std::unique_ptr<unsigned char, void (*)(void *)> stage((unsigned char *)dev_malloc((size_t)warps * stage_bytes), dev_free);
    for (int g = 0; g < G; g++) {
        KParams p = v->game_params(g);
        p.look.slot = v->looks[g].slot;
        p.env_first = g;
        p.env_step = G;
        p.env_count = per_game;
        p.look.list = base.look.list + g * per_game;
        p.look.count = &v->d_tickets->look_count;  // the list's count and the lookahead kernel's ticket
        p.look.stage = stage.get();
        p.look.stage_warps = warps;
        memset_async(p.look.count, 0, 2 * sizeof(unsigned int), v->stream);
        LaunchCtx lc = v->lctx();
        v->games[g]->lookahead_fill(p, lc);
    }
    v->sync();  // then the staging is released
    base.look.slot = v->looks[0].slot;  // last: VecEnv::step_shape reads a non-null slots pointer as lookahead on
    return 0;
}

int pgb200_level_lookahead_info(libenv_env *handle, int64_t *out) {
    VecEnv *v = (VecEnv *)handle;
    v->set_device();
    unsigned long long served[3] = {0, 0, 0};
    if (v->d_look_served) {
        if (!v->try_sync())
            return -1;
        copy_from_dev(served, v->d_look_served, sizeof(served));
    }
    for (int i = 0; i < 3; i++) out[i] = (int64_t)served[i];
    out[3] = v->look_bytes;
    return 0;
}

int pgb200_level_bank_info(libenv_env *handle, int *levels, int64_t *bytes) {
    VecEnv *v = (VecEnv *)handle;
    if (levels)
        *levels = v->bank_levels;
    if (bytes)
        *bytes = v->bank_bytes;
    return 0;
}

void pgb200_set_stream(libenv_env *handle, void *stream) {
    VecEnv *v = (VecEnv *)handle;
    v->set_device();
    const Stream next = (stream == PGB200_PRIVATE_STREAM) ? v->own_stream : (Stream)stream;
    // a stream that is capturing cannot be waited on, neither the new one nor the old one: moving into a
    // capture, the caller has ordered the handle's earlier work before the capture began
    if (!stream_capturing(next) && !v->capturing())
        v->sync();
    v->stream = next;
}

int pgb200_set_rgb_mirror(libenv_env *handle, void *mirror0, void *mirror1) {
#ifndef PG_HOSTSIM
    VecEnv *v = (VecEnv *)handle;
    v->set_device();
    if (!v->try_sync())
        return -1;
    v->mirror[0] = (uint8_t *)mirror0;
    v->mirror[1] = (uint8_t *)(mirror1 ? mirror1 : mirror0);
    v->mirror_parity = 0;
    return 0;
#else
    (void)handle; (void)mirror0; (void)mirror1;
    return -1;
#endif
}

int pgb200_set_consumer_output(libenv_env *handle, void *buffer, int dtype, int k_frames) {
#ifndef PG_HOSTSIM
    VecEnv *v = (VecEnv *)handle;
    v->set_device();
    if (!v->try_sync(true))
        return -1;
    if (buffer == nullptr || dtype == 0) {
        v->base.consumer = nullptr;
        return 0;
    }
    if ((dtype != 1 && dtype != 2) || k_frames < 1 || k_frames > 16)
        return -1;
    if (!v->d_consumer_lut)
        v->d_consumer_lut = v->alloc<uint16_t>(256);
    consumer_lut_kernel<<<1, 256, 0, v->stream>>>(v->d_consumer_lut, dtype == 2);
    CUDA_CHECK(cudaGetLastError());
    v->base.consumer = buffer;
    v->base.consumer_lut = v->d_consumer_lut;
    v->base.consumer_k = k_frames;
    v->consumer_slot = 0;
    v->consumer_steps = 0;
    memset_async(v->d_consumer_slot, 0, sizeof(int32_t), v->stream);
    // the current frame of every env becomes the newest frame of an otherwise empty stack
    for (size_t g = 0; g < v->games.size(); g++) {
        KParams p = v->game_params((int)g);
        p.env_first = (int)g;
        p.env_step = (int)v->games.size();
        p.env_count = v->num_envs / (int)v->games.size();
        LaunchCtx lc = v->lctx();
        v->games[g]->observe_only[v->view[g]](p, lc);
    }
    v->sync();
    return 0;
#else
    (void)handle; (void)buffer; (void)dtype; (void)k_frames;
    return -1;
#endif
}

int pgb200_debug_phase_offset(void) {
#ifdef PG_PHASE_TIMING
    return (int)offsetof(EnvHdr, dbg_phase);
#else
    return -1;
#endif
}

int pgb200_consumer_slot(libenv_env *handle) { return ((VecEnv *)handle)->consumer_slot; }

int pgb200_get_consumer_slot_device(libenv_env *handle, int32_t **out) {
#ifndef PG_HOSTSIM
    *out = ((VecEnv *)handle)->d_consumer_slot;
    return 0;
#else
    (void)handle;
    *out = nullptr;
    return -1;
#endif
}

int pgb200_mirror_parity(libenv_env *handle) { return ((VecEnv *)handle)->mirror_parity; }

void pgb200_act_device(libenv_env *handle) {
    VecEnv *v = (VecEnv *)handle;
    v->set_device();
    if (v->capturing()) {
#ifndef PG_HOSTSIM
        cudaStreamCaptureStatus st = cudaStreamCaptureStatusNone;
        if (cudaStreamIsCapturing(v->stream, &st) == cudaErrorStreamCaptureImplicit) {
            cudaGetLastError();
            pg_fatal("pgb200_act_device: a CUDA graph capture is running on another stream and the handle is on the legacy "
                     "default stream; rebind it to the capturing stream first (pgb200_set_stream)\n");
        }
        if (v->timing)
            pg_fatal("pgb200_act_device: a step under kernel timing cannot be captured\n");
#endif
        // what a captured step cannot contain: the initial reset, host-side state that changes from step to
        // step (the mirror parity, the host buffers' copies) and the timing events
        if (!v->initial_reset_done)
            pg_fatal("pgb200_act_device: the initial reset cannot be captured; call pgb200_get_device_buffers first\n");
        if (v->mirror[0])
            pg_fatal("pgb200_act_device: a step with the peer mirror set cannot be captured\n");
        if (v->have_host_bufs)
            pg_fatal("pgb200_act_device: a handle with host buffers cannot be captured\n");
    }
    v->ensure_initial_reset();
    v->launch(false);
}

void pgb200_sync(libenv_env *handle) {
    VecEnv *v = (VecEnv *)handle;
    v->set_device();
    v->refuse_in_capture("pgb200_sync");
    v->sync();
}

uint32_t pgb200_get_errors(libenv_env *handle, uint32_t *host_out) {
    VecEnv *v = (VecEnv *)handle;
    v->set_device();
    if (!v->try_sync())
        return UINT32_MAX;
    const size_t N = (size_t)v->num_envs;
    std::vector<EnvHdr> hdr(N);
    copy_from_dev(hdr.data(), v->base.hdr, N * sizeof(EnvHdr));
    uint32_t any = 0;
    for (size_t e = 0; e < N; e++) {
        if (host_out)
            host_out[e] = hdr[e].err;
        any |= hdr[e].err;
    }
    return any;
}

int pgb200_debug_cycles(libenv_env *handle, uint32_t *host_out) {
    VecEnv *v = (VecEnv *)handle;
    if (!v->base.dbg_cycles)
        return -1;
    v->set_device();
    if (!v->try_sync())
        return -1;
    copy_from_dev(host_out, v->base.dbg_cycles, (size_t)v->num_envs * 4);
    return 0;
}

int pgb200_debug_read_env(libenv_env *handle, int env, void *hdr_out, void *ents_out, int max_ents) {
    VecEnv *v = (VecEnv *)handle;
    if (env < 0 || env >= v->num_envs)
        return -1;
    v->set_device();
    if (!v->try_sync())
        return -1;
    EnvHdr hdr;
    const KParams &p = v->base;
    copy_from_dev(&hdr, p.hdr + env, sizeof(EnvHdr));
    if (hdr_out)
        memcpy(hdr_out, &hdr, sizeof(EnvHdr));
    int n = hdr.n_ents < max_ents ? hdr.n_ents : max_ents;
    if (ents_out && n > 0)
        copy_from_dev(ents_out, p.ents + (size_t)env * p.ent_stride, (size_t)n * sizeof(Entity));
    return hdr.n_ents;
}

// ---- get_state / set_state (vecgame.cpp:437-457) and their batched forms
//
// A transfer moves each listed env's packed record (StateSlot, pg_kernels.cuh) through the handle's staging, in chunks
// that fit it: first the headers, which size the records, then the records, with one copy each way per chunk. The host
// writes and reads the blobs from those records with io_env (pg_state_io.h); the device only gathers and scatters them.
}  // extern "C"

namespace {

constexpr size_t kStateStageBudget = (size_t)256 << 20;  // staging a transfer may grow to, device and pinned each

size_t align16(size_t n) { return (n + 15) & ~(size_t)15; }

// env's slot for the header h: its live entities and cells, bounded by the handle's capacities, and its game's
// persistent scratch words (the ones io_tail reads, and dodgeball's rooms)
StateSlot state_slot(const VecEnv *v, int env, const EnvHdr &h) {
    const KParams &p = v->base;
    const GameVTable *g = v->games[(size_t)env % v->games.size()];
    StateSlot s{};
    s.env = env;
    s.n_ents = std::min(std::max(h.n_ents, 0), p.ent_stride - 1);
    s.cells = (int)std::min<int64_t>(std::max<int64_t>((int64_t)h.main_width * h.main_height, 0), p.grid_stride);
    s.scratch_first = g->persist_scratch_first;
    s.scratch_words = g->persist_scratch_words;
    return s;
}

// The headers of envs[0, n)
std::vector<EnvHdr> gather_headers(VecEnv *v, const int32_t *envs, int n) {
    std::vector<EnvHdr> hdrs((size_t)n);
    const int chunk = (int)std::min<size_t>((size_t)n, (kStateStageBudget - 16) / (sizeof(int32_t) + sizeof(EnvHdr)));
    v->grow_state_stage(align16((size_t)chunk * sizeof(int32_t)) + (size_t)chunk * sizeof(EnvHdr));
    for (int i0 = 0; i0 < n; i0 += chunk) {
        const int k = std::min(chunk, n - i0);
        const size_t hdrs_off = align16((size_t)k * sizeof(int32_t));
        const int32_t *d_envs = reinterpret_cast<const int32_t *>(v->d_state_stage);
        EnvHdr *d_hdrs = reinterpret_cast<EnvHdr *>(v->d_state_stage + hdrs_off);
        memcpy(v->h_state_stage, envs + i0, (size_t)k * sizeof(int32_t));
        copy_to_dev_async(v->d_state_stage, v->h_state_stage, (size_t)k * sizeof(int32_t), v->stream);
#ifndef PG_HOSTSIM
        state_headers_kernel<<<(k + 3) / 4, 128, 0, v->stream>>>(v->base.hdr, d_envs, k, d_hdrs);
        CUDA_CHECK(cudaGetLastError());
#else
        for (int i = 0; i < k; i++) bank_copy_vecs(d_hdrs + i, v->base.hdr + d_envs[i], (int)sizeof(EnvHdr));
#endif
        copy_from_dev_async(v->h_state_stage + hdrs_off, d_hdrs, (size_t)k * sizeof(EnvHdr), v->stream);
        v->sync();
        memcpy(static_cast<void *>(hdrs.data() + i0), v->h_state_stage + hdrs_off, (size_t)k * sizeof(EnvHdr));
    }
    return hdrs;
}

// The packed records of slots[0, n), in chunks that fit the staging: the slots of a chunk get their offsets in it, and
// f(i0, k, recs) runs for its slots [i0, i0 + k) with their records at recs (the pinned staging). STORE false: the
// records are gathered from the envs and copied down before f reads them. STORE true: f writes them, and they are
// copied up and scattered into the envs.
template <bool STORE, class F>
void move_records(VecEnv *v, std::vector<StateSlot> &slots, F &&f) {
    const int n = (int)slots.size();
    size_t total = align16((size_t)n * sizeof(StateSlot));
    for (const StateSlot &s : slots) total += state_record_bytes(s);
    v->grow_state_stage(std::min(total, kStateStageBudget));
    for (int i0 = 0; i0 < n;) {
        int k = 0;
        size_t rec_bytes = 0;
        for (; i0 + k < n; k++) {
            const size_t bytes = state_record_bytes(slots[i0 + k]);
            if (k > 0 && align16((size_t)(k + 1) * sizeof(StateSlot)) + rec_bytes + bytes > v->state_stage_bytes)
                break;
            slots[i0 + k].offset = (int64_t)rec_bytes;
            rec_bytes += bytes;
        }
        const size_t recs_off = align16((size_t)k * sizeof(StateSlot));
        const StateSlot *d_slots = reinterpret_cast<const StateSlot *>(v->d_state_stage);
        unsigned char *h_recs = v->h_state_stage + recs_off, *d_recs = v->d_state_stage + recs_off;
        memcpy(static_cast<void *>(v->h_state_stage), slots.data() + i0, (size_t)k * sizeof(StateSlot));
        if (STORE)
            f(i0, k, h_recs);
        copy_to_dev_async(v->d_state_stage, v->h_state_stage, STORE ? recs_off + rec_bytes : (size_t)k * sizeof(StateSlot), v->stream);
#ifndef PG_HOSTSIM
        state_records_kernel<STORE><<<(k + 3) / 4, 128, 0, v->stream>>>(v->base, d_slots, k, d_recs);
        CUDA_CHECK(cudaGetLastError());
#else
        for (int i = 0; i < k; i++) state_move<STORE>(v->base, d_slots[i], d_recs + d_slots[i].offset);
#endif
        if (!STORE)
            copy_from_dev_async(h_recs, d_recs, rec_bytes, v->stream);
        v->sync();  // the pinned staging is free for the next chunk
        if (!STORE)
            f(i0, k, h_recs);
        i0 += k;
    }
}

// The packed record `rec` of slot s into the HostEnv io_env works on (PACK false), or back out of it (PACK true)
template <bool PACK>
void state_host_move(const StateSlot &s, host::HostEnv &e, unsigned char *rec) {
    auto part = [&](void *env_part, size_t off, size_t bytes) {
        if (bytes == 0)
            return;
        if (PACK)
            memcpy(rec + off, env_part, bytes);
        else
            memcpy(env_part, rec + off, bytes);
    };
    part(&e.h, 0, sizeof(EnvHdr));
    part(&e.rng, sizeof(EnvHdr), sizeof(MT19937));
    part(&e.lvl_rng, sizeof(EnvHdr) + sizeof(MT19937), sizeof(MT19937));
    part(e.ents.data(), state_ents_off(), (size_t)s.n_ents * sizeof(Entity));
    part(e.grid.data(), state_grid_off(s), (size_t)s.cells * sizeof(int16_t));
    part(e.scratch.data() + s.scratch_first, state_scratch_off(s), (size_t)s.scratch_words * sizeof(int32_t));
}

// f(i, t) for every i in [0, n) on `threads` threads, the calling one included (t: the thread's index). Once all have
// finished, the exception of the lowest i that threw, if any, is thrown again.
template <class F>
void parallel_for(int n, int threads, F &&f) {
    std::atomic<int> next{0};
    std::mutex m;
    int first_bad = n;
    std::exception_ptr err;
    auto work = [&](int t) {
        for (int i; (i = next.fetch_add(1)) < n;) {
            try {
                f(i, t);
            } catch (...) {
                std::lock_guard<std::mutex> lock(m);
                if (i < first_bad) {
                    first_bad = i;
                    err = std::current_exception();
                }
            }
        }
    };
    std::vector<std::thread> pool;
    for (int t = 1; t < threads; t++) pool.emplace_back(work, t);
    work(0);
    for (std::thread &th : pool) th.join();
    if (err)
        std::rethrow_exception(err);
}

// Host threads a transfer of n envs writes or reads its blobs on: the text form of three generators makes a blob cost
// the host far more than its bytes cost the copies (DESIGN §7)
int state_threads(int n) {
    const int cores = (int)std::max(1u, std::thread::hardware_concurrency());
    return std::max(1, std::min({cores, 32, n / 16}));
}

// Hands the records of envs[0, n) to f(i, slot, e, t) as the HostEnv e that io_env reads and writes, on
// state_threads(n) threads (t: the thread's index, e its own), then chunk_done(i0, k) on the calling thread once the envs
// [i0, i0 + k) of a chunk are done. The parts of e outside the env's packed record hold what an earlier env left
// there: io_env neither reads them nor writes anything there that is stored back.
template <class F, class Done>
void gather_states(VecEnv *v, const int32_t *envs, int n, F &&f, Done &&chunk_done) {
    const std::vector<EnvHdr> hdrs = gather_headers(v, envs, n);
    std::vector<StateSlot> slots((size_t)n);
    for (int i = 0; i < n; i++) slots[i] = state_slot(v, envs[i], hdrs[i]);
    const int threads = state_threads(n);
    std::vector<host::HostEnv> es((size_t)threads);
    for (host::HostEnv &e : es) {
        e.ent_cap = v->base.ent_stride - 1;
        e.ents.resize((size_t)v->base.ent_stride);
        e.grid.resize((size_t)v->base.grid_stride);
        e.scratch.resize((size_t)v->base.scratch_stride);
    }
    move_records<false>(v, slots, [&](int i0, int k, unsigned char *recs) {
        parallel_for(k, std::min(threads, k), [&](int j, int t) {
            const StateSlot &s = slots[(size_t)(i0 + j)];
            state_host_move<false>(s, es[t], recs + s.offset);
            f(i0 + j, s, es[t], t);
        });
        chunk_done(i0, k);
    });
}

// env's blob, written into data[0, length); returns its size. A too small buffer throws, and is fatal for the caller,
// like the reference's fassert.
int serialize_state(const VecEnv *v, int env, const host::HostEnv &e, char *data, size_t length) {
    const GameVTable *g = v->games[(size_t)env % v->games.size()];
    host::WriteBuf b(data, length);
    host::serialize_env(g->name, g->id, e, v->const_fields, b);
    return (int)b.offset;
}

// Game::observe of the envs listed per game, on the handle's stream: game g's are the first *(counts + g) of
// lists + first[g], a count read on the device and at most bound[g], which sizes the list camera's grid. One
// launch_observe_list per game with bound[g] > 0.
void observe_lists(VecEnv *v, int32_t *lists, unsigned int *counts, const std::vector<size_t> &first, const std::vector<uint32_t> &bound) {
    for (size_t g = 0; g < v->games.size(); g++) {
        if (bound[g] == 0)
            continue;
        KParams p = v->game_params((int)g);
        p.reset_list = lists + first[g];
        p.reset_count = counts + g;
        p.env_count = (int)bound[g];
        LaunchCtx lc = v->lctx();
        v->games[g]->observe_list[v->view[g]](p, lc);
    }
}

// Game::observe of envs[0, n) (distinct, the handle's stream idle): one launch_observe_list per game with listed envs
void observe_states(VecEnv *v, const int32_t *envs, int n) {
    const size_t G = v->games.size();
    std::vector<uint32_t> counts(G, 0);
    for (int i = 0; i < n; i++) counts[(size_t)envs[i] % G]++;
    // staging: the per-game counts, then the per-game lists one after the other
    const size_t lists_off = align16(G * sizeof(uint32_t));
    v->grow_state_stage(lists_off + (size_t)n * sizeof(int32_t));
    std::vector<size_t> first(G, 0), next(G);
    for (size_t g = 1; g < G; g++) first[g] = first[g - 1] + counts[g - 1];
    next = first;
    int32_t *h_lists = reinterpret_cast<int32_t *>(v->h_state_stage + lists_off);
    for (int i = 0; i < n; i++) h_lists[next[(size_t)envs[i] % G]++] = envs[i];
    memcpy(v->h_state_stage, counts.data(), G * sizeof(uint32_t));
    copy_to_dev_async(v->d_state_stage, v->h_state_stage, lists_off + (size_t)n * sizeof(int32_t), v->stream);
    observe_lists(v, reinterpret_cast<int32_t *>(v->d_state_stage + lists_off), reinterpret_cast<unsigned int *>(v->d_state_stage),
                  first, counts);
    v->sync();
    v->rgb_copy_enqueued = false;  // a DMA started behind the last step predates these frames: observe copies again
}

// set_state of envs[0, n) (distinct, in range; the handle's stream idle) from the blobs data[offsets[i], offsets[i + 1]).
// Every blob is read, onto the env's gathered records (deserialize_env keeps what the blob does not carry), before any
// env changes; then the restored records are scattered and the envs observed.
void load_states(VecEnv *v, const int32_t *envs, int n, const char *data, const int64_t *offsets) {
    std::vector<StateSlot> slots((size_t)n);
    std::vector<std::vector<unsigned char>> records((size_t)n);  // the restored packed records
    try {
        gather_states(
            v, envs, n,
            [&](int i, const StateSlot &, host::HostEnv &e, int) {
                const int env = envs[i];
                const GameVTable *g = v->games[(size_t)env % v->games.size()];
                try {
                    host::ReadBuf b(data + offsets[i], (size_t)std::max<int64_t>(offsets[i + 1] - offsets[i], 0));
                    host::deserialize_env(g->name, g->id, e, b);
                } catch (const std::exception &ex) {
                    throw std::runtime_error(std::string(ex.what()) + " (env " + std::to_string(env) + ")");
                }
                slots[i] = state_slot(v, env, e.h);
                records[i].resize(state_record_bytes(slots[i]));
                state_host_move<true>(slots[i], e, records[i].data());
            },
            [](int, int) {});
    } catch (const std::exception &ex) {
        pg_fatal("set_state: %s\n", ex.what());
    }
    move_records<true>(v, slots, [&](int i0, int k, unsigned char *recs) {
        for (int i = i0; i < i0 + k; i++) memcpy(recs + slots[i].offset, records[i].data(), records[i].size());
    });
    observe_states(v, envs, n);
}

}  // namespace

extern "C" {

int pgb200_get_states(libenv_env *handle, const int32_t *envs, int n, const char **data, const int64_t **offsets) {
    VecEnv *v = (VecEnv *)handle;
    v->set_device();
    if (n < 0 || (n > 0 && !envs) || !data || !offsets)
        return -1;
    for (int i = 0; i < n; i++)
        if (envs[i] < 0 || envs[i] >= v->num_envs)
            return -1;
    if (!v->try_sync(true))  // wait_for_stepping_threads
        return -1;
    v->state_blobs.clear();
    v->state_offsets.assign(1, 0);
    std::vector<std::vector<char>> scratch((size_t)state_threads(n));  // per thread
    std::vector<std::string> blobs((size_t)n);                          // of the chunk in flight
    try {
        gather_states(
            v, envs, n,
            [&](int i, const StateSlot &s, const host::HostEnv &e, int t) {
                // a blob takes at most twice its record (four bytes per grid cell) and the text of three generators
                std::vector<char> &buf = scratch[(size_t)t];
                buf.resize(std::max(buf.size(), ((size_t)64 << 10) + 2 * state_record_bytes(s)));
                blobs[(size_t)i].assign(buf.data(), (size_t)serialize_state(v, envs[i], e, buf.data(), buf.size()));
            },
            [&](int i0, int k) {
                for (int i = i0; i < i0 + k; i++) {
                    v->state_blobs.insert(v->state_blobs.end(), blobs[(size_t)i].begin(), blobs[(size_t)i].end());
                    v->state_offsets.push_back((int64_t)v->state_blobs.size());
                    std::string().swap(blobs[(size_t)i]);
                }
            });
    } catch (const std::exception &ex) {
        pg_fatal("get_state: %s\n", ex.what());
    }
    *data = v->state_blobs.data();
    *offsets = v->state_offsets.data();
    return 0;
}

int pgb200_set_states(libenv_env *handle, const int32_t *envs, int n, const char *data, const int64_t *offsets) {
    VecEnv *v = (VecEnv *)handle;
    v->set_device();
    if (n < 0 || (n > 0 && (!envs || !data || !offsets)))
        return -1;
    std::vector<uint8_t> listed((size_t)v->num_envs, 0);
    for (int i = 0; i < n; i++) {
        if (envs[i] < 0 || envs[i] >= v->num_envs || listed[(size_t)envs[i]])
            return -1;
        listed[(size_t)envs[i]] = 1;
    }
    if (!v->try_sync(true))
        return -1;
    load_states(v, envs, n, data, offsets);
    return 0;
}

int get_state(libenv_env *handle, int env_idx, char *data, int length) {
    VecEnv *v = (VecEnv *)handle;
    v->set_device();
    pg_fassert(env_idx >= 0 && env_idx < v->num_envs);
    if (!v->try_sync(true))  // wait_for_stepping_threads
        return -1;
    int len = 0;
    try {
        gather_states(
            v, &env_idx, 1,
            [&](int, const StateSlot &, const host::HostEnv &e, int) {
                len = serialize_state(v, env_idx, e, data, (size_t)(length < 0 ? 0 : length));
            },
            [](int, int) {});
    } catch (const std::exception &ex) {
        pg_fatal("get_state: %s\n", ex.what());
    }
    return len;
}

void set_state(libenv_env *handle, int env_idx, char *data, int length) {
    VecEnv *v = (VecEnv *)handle;
    v->set_device();
    pg_fassert(env_idx >= 0 && env_idx < v->num_envs);
    v->refuse_in_capture("set_state");
    v->ensure_initial_reset();
    v->sync();
    const int64_t offsets[2] = {0, length < 0 ? 0 : length};
    load_states(v, &env_idx, 1, data, offsets);
}

// ---- snapshot slots (SnapshotStore, pg_kernels.cuh). One allocation holds the caller's arrays, the load list, the
// per-game table and the slots, each part 16-byte aligned.
int pgb200_get_snapshots(libenv_env *handle, int slots, struct pgb200_snapshots *out) {
    VecEnv *v = (VecEnv *)handle;
    v->set_device();
    SnapshotStore &st = v->snaps;
    if (!out || slots < 1 || (st.slots && slots != st.count))
        return -1;
    if (!st.slots) {
        const KParams &p = v->base;
        const size_t G = v->games.size(), N = (size_t)v->num_envs, S = (size_t)slots;
        StateSlot widest{};
        widest.n_ents = p.ent_stride - 1;
        widest.cells = p.grid_stride;
        for (const GameVTable *g : v->games) widest.scratch_words = std::max(widest.scratch_words, g->persist_scratch_words);
        const size_t slot_bytes = kSnapshotRecordOff + state_record_bytes(widest);
        const size_t source_off = align16(S * sizeof(int32_t)), load_off = source_off + align16(S * sizeof(int32_t));
        const size_t list_off = load_off + align16(N * sizeof(int32_t)), counts_off = list_off + align16(N * sizeof(int32_t));
        const size_t persist_off = counts_off + align16(G * sizeof(uint32_t)), slots_off = persist_off + align16(2 * G * sizeof(int32_t));
        if (S > ((size_t)INT64_MAX - slots_off) / slot_bytes)
            return -1;
        const size_t bytes = slots_off + S * slot_bytes;
        if (v->capturing())  // the allocation and the fills below would invalidate the caller's capture
            return -1;
        unsigned char *mem = (unsigned char *)dev_try_malloc(bytes);
        if (!mem)
            return -1;
        v->owned_dev.push_back(mem);
        v->ensure_initial_reset();
        std::vector<int32_t> persist;
        for (const GameVTable *g : v->games) persist.insert(persist.end(), {g->persist_scratch_first, g->persist_scratch_words});
        memset_async(mem, 0xff, list_off, v->stream);  // save_from, source and load_from: every entry -1
        copy_to_dev_async(mem + persist_off, persist.data(), persist.size() * sizeof(int32_t), v->stream);
        v->sync();
        st.slot_bytes = (int64_t)slot_bytes;
        st.count = slots;
        st.num_envs = v->num_envs;
        st.games = (int32_t)G;
        st.save_from = reinterpret_cast<int32_t *>(mem);
        st.source = reinterpret_cast<int32_t *>(mem + source_off);
        st.load_from = reinterpret_cast<int32_t *>(mem + load_off);
        st.list = reinterpret_cast<int32_t *>(mem + list_off);
        st.counts = reinterpret_cast<unsigned int *>(mem + counts_off);
        st.persist = reinterpret_cast<const int32_t *>(mem + persist_off);
        st.slots = mem + slots_off;  // last: pgb200_apply_snapshots reads a non-null slots pointer as the store
        v->snap_bytes = (int64_t)bytes;
    }
    out->save_from = st.save_from;
    out->load_from = st.load_from;
    out->source = st.source;
    out->bytes = v->snap_bytes;
    return 0;
}

int pgb200_apply_snapshots(libenv_env *handle) {
    VecEnv *v = (VecEnv *)handle;
    v->set_device();
    const SnapshotStore &st = v->snaps;
    if (!st.slots)
        return -1;
    const size_t G = v->games.size();
    memset_async(st.counts, 0, G * sizeof(uint32_t), v->stream);
#ifndef PG_HOSTSIM
    snapshot_save_kernel<<<(st.count + 3) / 4, 128, 0, v->stream>>>(v->base, st);
    CUDA_CHECK(cudaGetLastError());
    snapshot_load_kernel<<<(st.num_envs + 3) / 4, 128, 0, v->stream>>>(v->base, st);
    CUDA_CHECK(cudaGetLastError());
#else
    for (int s = 0; s < st.count; s++) snapshot_save(v->base, st, s);
    for (int env = 0; env < st.num_envs; env++) snapshot_load(v->base, st, env);
#endif
    v->launches += 2;
    // each game's segment of the list: its envs are at most num_envs / G
    std::vector<size_t> first(G);
    for (size_t g = 0; g < G; g++) first[g] = g * (size_t)(st.num_envs / st.games);
    observe_lists(v, st.list, st.counts, first, std::vector<uint32_t>(G, (uint32_t)(st.num_envs / st.games)));
    v->rgb_copy_enqueued = false;  // a DMA started behind the last step predates the loaded envs' frames
    return 0;
}

int pgb200_frame_info(const char *game, int *frame_bytes, int *ctas_per_sm) {
    const GameVTable *g = find_game(game);
    if (!g)
        return -1;
    *frame_bytes = g->frame_bytes[0];
    *ctas_per_sm = g->render_ctas_per_sm[0];
    return 0;
}

int64_t pgb200_kernel_launches(libenv_env *handle) { return ((VecEnv *)handle)->launches; }

void pgb200_set_launch_shape(libenv_env *handle, int chunks, int serialize) {
    VecEnv *v = (VecEnv *)handle;
    v->set_device();
    v->refuse_in_capture("pgb200_set_launch_shape");
    v->sync();
    v->force_chunks = chunks;
    v->serialize_launches = serialize != 0;
}

int pgb200_kernel_timing_begin(libenv_env *handle, int max_launch_pairs) {
#ifndef PG_HOSTSIM
    VecEnv *v = (VecEnv *)handle;
    v->set_device();
    // a step with final outputs renders in both of its phases, which one quadruple of events cannot time
    if (v->step_shape(false).final_outputs || !v->try_sync())
        return -1;
    while ((int)v->tev_pool.size() < 4 * max_launch_pairs) {
        cudaEvent_t e;
        CUDA_CHECK(cudaEventCreate(&e));
        v->tev_pool.push_back(v->own(e));
    }
    v->tev_used = 0;
    v->tev_envs.clear();
    v->timing = true;
    return 0;
#else
    return -1;
#endif
}

int pgb200_kernel_timing_end(libenv_env *handle, double *out) {
#ifndef PG_HOSTSIM
    VecEnv *v = (VecEnv *)handle;
    v->set_device();
    if (!v->try_sync())
        return -1;
    v->timing = false;
    double logic_ms = 0, setup_ms = 0, render_ms = 0, envs = 0;
    const int pairs = (int)(v->tev_used / 4);
    for (int i = 0; i < pairs; i++) {
        float a = 0, b = 0, c2 = 0;
        CUDA_CHECK(cudaEventElapsedTime(&a, v->tev_pool[4 * i], v->tev_pool[4 * i + 1]));
        CUDA_CHECK(cudaEventElapsedTime(&b, v->tev_pool[4 * i + 1], v->tev_pool[4 * i + 2]));
        CUDA_CHECK(cudaEventElapsedTime(&c2, v->tev_pool[4 * i + 2], v->tev_pool[4 * i + 3]));
        logic_ms += a;
        setup_ms += b;
        render_ms += c2;
        envs += v->tev_envs[i];
    }
    out[0] = logic_ms;
    out[1] = render_ms;
    out[2] = pairs;
    out[3] = envs;
    out[4] = setup_ms;
    v->tev_used = 0;
    v->tev_envs.clear();
    return pairs;
#else
    return -1;
#endif
}

}  // extern "C"
