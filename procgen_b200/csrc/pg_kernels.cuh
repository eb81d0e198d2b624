// Per-env work items (logic phase, render phases) and the launch parameter block. The CUDA
// kernels in pg_runtime.cu are thin wrappers that map one CTA to one env and put barriers between
// the phases; the CPU debug harness runs the very same phase functions in plain loops.
#pragma once
#include "pg_raster.cuh"

namespace pg {

// A handle's rollout (pgb200_get_rollout): `slots` copies of the step outputs rgb, rew and first, slot-major
struct Rollout {
    uint8_t *rgb;      // [slots][num_envs][64][64][3]
    float *rew;        // [slots][num_envs]
    uint8_t *first;    // [slots][num_envs]
    int32_t *cursor;   // [1] the slot the current step writes (device)
    int32_t slots;
    int32_t num_envs;  // the handle's, not the launch's
};

struct KParams {
    // state (HBM)
    EnvHdr *hdr;
    Entity *ents;
    int16_t *grid;
    MT19937 *rng;
    MT19937 *lvl_rng;
    int32_t *scratch;
    RotBlit *rot_scratch;       // [N][rot_stride] rotated-sprite / span records
    Blit *blit_list;            // [N][blit_stride] background-less blit lists (entities in draw order, then overlays)
    unsigned char *frame_setup; // [N][frame_setup_stride bytes] FrameSharedT of the env's game (setup kernel -> render kernel)
    Blit *cell_spill;           // [N][cell_spill_stride] general cell blits that do not fit the render CTA's shared memory
    const GameAssets *assets;   // table of the game this launch handles
    const uint32_t *atlas;
    TileTable tiles;            // pre-scaled cell tiles of every sprite (texels == nullptr: disabled)
    // libenv-visible buffers (vecgame.cpp:212-268), one slot per env
    const int32_t *action;
    uint8_t *rgb;               // [N][64][64][3]
    float *rew;
    uint8_t *first;
    int32_t *info_prev_level_seed;
    uint8_t *info_prev_level_complete;
    int32_t *info_level_seed;
    const uint32_t *lvl_seeds;  // per-env seed for level_seed_rand_gen (vecgame.cpp:301-314)
    int32_t *next_level_seed;   // optional [N] caller-chosen seed of the env's next level, -1 = none; null = off
    // strides (elements)
    int32_t ent_stride;         // ent_cap + 1 (ghost slot)
    int32_t grid_stride;
    int32_t scratch_stride;
    int32_t rot_stride;
    int32_t blit_stride;
    int32_t frame_setup_stride;
    int32_t cell_spill_stride;
    // which envs this launch covers: env = env_first + i * env_step, i in [0, env_count)
    int32_t env_first, env_step, env_count;
    // construction-time options (game.cpp:42-75, vecgame.cpp:284-293)
    Options options;
    int32_t level_seed_low, level_seed_high;
    int32_t game_id;
    int32_t fixed_asset_seed;   // FNV-1a of the game name (vecgame.cpp:156-167, 324-327)
    int32_t snap;
    int32_t env_global_offset;  // game_n = env_global_offset + env
    // optional second output for on-device learners (SURVEY §8(f)4): normalised fp16 / bf16, planar
    // CHW, k-frame stack kept as a 2k-slot ring so that the ordered stack is always one contiguous view
    void *consumer;             // [N][slots][3][64][64] 16-bit elements; null = off
    const uint16_t *consumer_lut;  // [256] = (16-bit float)(v / 255.f)
    int32_t consumer_k;         // frames per stack; slots = k == 1 ? 1 : 2k
    const int32_t *consumer_slot_dev;  // device: ring position this step writes, t mod k (advanced on the device once per step)
    uint32_t *dbg_cycles;       // optional [N] per-env logic duration in SM cycles (profiling aid)
    // optional final outputs (pgb200_get_final_outputs); null = off. A step then runs in two phases per launch:
    // A renders the final state of the envs whose level ends, B resets exactly those (reset_list) and renders again
    uint8_t *final_rgb;         // [N][64][64][3]
    uint8_t *level_end;         // [N] why env's level ended in this step (PGB200_LEVEL_END_*), 0 = it did not
    int32_t *reset_list;        // this launch's own segment of an [N] list: the envs phase B resets
    unsigned int *reset_count;  // entries in reset_list (device; a word of the launch's TicketSlot)
    // optional pause mask (pgb200_get_pause_mask); null = off. Only the logic kernel reads the caller's array: it
    // records each env's decision in `paused`, which the step's setup and render kernels read, so that every kernel
    // of one step agrees even if the caller rewrites the mask while the step runs
    const uint8_t *pause;       // [N] caller's mask: != 0 = env does not step
    uint8_t *paused;            // [N] handle-owned: env is paused in the current step
    // optional level bank (pgb200_build_level_bank); bank.slots null = off. The launch's game's slots. A banked
    // handle steps in two phases as with final outputs; without them, phase A's level_end goes to bank_level_end
    LevelBank bank;
    uint8_t *bank_level_end;    // [N] handle-owned
    // optional level lookahead (pgb200_enable_level_lookahead); look.slot.slots null = off. The handle then steps in
    // two phases as with a bank, and its phase B lists the envs whose next level the lookahead kernel generates
    LevelLookahead look;
    // optional rollout (pgb200_get_rollout); roll.rgb null = off. Every step also stores each env's rgb, rew and first
    // into slot *roll.cursor of the ring, which the step advances on the device before its render kernels
    Rollout roll;
    // optional action repeat (pgb200_get_action_repeat); null = off. Only the logic kernel reads it: env plays up to
    // max(repeat[env], 1) game steps per step, and stops after the first whose level ends
    const int32_t *repeat;      // [N] caller's repeat counts
};

// Where env's outputs of the current step go in the rollout: slot *roll.cursor, slot-major
PG_HD size_t rollout_index(const KParams &p, int env) { return (size_t)*p.roll.cursor * (size_t)p.roll.num_envs + (size_t)env; }

// The rollout's copy of env's scalar outputs of this step, which the logic or finish kernel has written by the time a
// frame of the step is rendered
PG_HD void rollout_store_scalars(const KParams &p, int env) {
    const size_t i = rollout_index(p, env);
    p.roll.rew[i] = p.rew[env];
    p.roll.first[i] = p.first[env];
}

// env's rollout slot of this step gets its current rgb, rew and first, copied by `lane` of `nlanes` threads (the CTA
// of a paused env; one thread in the host debug build, behind each rendered frame)
PG_HD void rollout_copy_frame(const KParams &p, int env, int lane, int nlanes) {
    constexpr int kFrameVecs = RES_W * RES_H * 3 / 16;
    const BankVec *src = reinterpret_cast<const BankVec *>(p.rgb) + (size_t)env * kFrameVecs;
    BankVec *dst = reinterpret_cast<BankVec *>(p.roll.rgb) + rollout_index(p, env) * kFrameVecs;
    for (int w = lane; w < kFrameVecs; w += nlanes) dst[w] = src[w];
    if (lane == 0)
        rollout_store_scalars(p, env);
}

// Whether env's frame in render pass PASS is the final frame of its level: pass 1 (phase A of a step with final
// outputs) of an env whose level ended. It goes to final_rgb, and neither the consumer output nor the rollout gets it.
template <int PASS>
PG_HD bool is_final_frame(const KParams &p, int env) { return PASS == 1 && p.level_end[env] != 0; }

// If `when`, appends env to `list`, whose length is *count: on the device the calling warp's lane 0 does. The list and
// its count are read only to append (the logic kernel's stack frame depends on it).
PG_HD void list_append(bool when, int32_t *const &list, unsigned int *const &count, int env) {
#if defined(__CUDA_ARCH__)
    if (when && (threadIdx.x & 31u) == 0)
        list[atomicAdd(count, 1u)] = env;
#else
    if (when)
        list[(*count)++] = env;
#endif
}

PG_HD Ctx make_ctx(const KParams &p, int env) {
    Ctx c;
    c.h = p.hdr + env;
    c.ents = p.ents + (size_t)env * p.ent_stride;
    c.grid = p.grid + (size_t)env * p.grid_stride;
    c.rng = p.rng + env;
    c.lvl_rng = p.lvl_rng + env;
    c.assets = p.assets;
    c.scratch = p.scratch + (size_t)env * p.scratch_stride;
    c.ent_cap = p.ent_stride - 1;
    c.grid_cap = p.grid_stride;
    c.scratch_cap = p.scratch_stride;
    c.obst_hi = -1;
    c.rot_scratch_raw = (p.rot_scratch && p.rot_stride > 0) ? (void *)(p.rot_scratch + (size_t)env * p.rot_stride) : nullptr;
    c.blit_list = p.blit_list ? p.blit_list + (size_t)env * p.blit_stride : nullptr;
    c.cell_spill = p.cell_spill ? p.cell_spill + (size_t)env * p.cell_spill_stride : nullptr;
    ctx_refresh(c);
    return c;
}

// Game::observe's scalar stores (game.cpp:160-164)
PG_HD void write_step_outputs(const KParams &p, int env, const EnvHdr &h) {
    p.rew[env] = h.reward;
    p.first[env] = (uint8_t)(h.done != 0);
    p.info_prev_level_seed[env] = h.prev_level_seed;
    p.info_prev_level_complete[env] = (uint8_t)(h.level_complete != 0);
    p.info_level_seed[env] = h.current_level_seed;
}

// Construction + first reset (VecGame ctor per-env part vecgame.cpp:309-330, then
// set_buffers -> reset(); observe(), vecgame.cpp:349-353). One thread.
template <class G, class Frame>
PG_HD void env_init_logic(const KParams &p, int env) {
    Ctx c = make_ctx(p, env);
    G::init_constants(c);
    ctx_refresh(c);
    EnvHdr &h = *c.h;
    h.options = p.options;
    h.game_id = p.game_id;
    h.fixed_asset_seed = p.fixed_asset_seed;
    h.game_n = p.env_global_offset + env;
    h.level_seed_low = p.level_seed_low;
    h.level_seed_high = p.level_seed_high;
    mt_seed(*c.lvl_rng, p.lvl_seeds[env]);
    c.rng->seeded = 0;
    Engine<G>::reset(c);
    h.initial_reset_complete = 1;
    Raster<G, Frame>::prepare_camera(c);
    write_step_outputs(p, env, h);
}

// Game::observe without a step (set_state, vecgame.cpp:454-456): the camera and the scalar outputs (game.cpp:160-164).
// One thread.
template <class G, class Frame>
PG_HD void env_observe(const KParams &p, int env) {
    Ctx c = make_ctx(p, env);
    Raster<G, Frame>::prepare_camera(c);
    write_step_outputs(p, env, *c.h);
}

// ---- state transfers (get_state / set_state and their batched forms). The device moves, per listed env, exactly the
// part of its records that the state blob is written from or read into (pg_state_io.h io_env): the header, both
// generators, the live entities, the main_width x main_height grid cells and the game's persistent scratch words. They
// travel as one packed record per env, each part 16-byte aligned:
//   EnvHdr | rand_gen | level_seed_rand_gen | Entity[n_ents] | int16 grid[cells] | int32 scratch[scratch_words]
// The host serializes from and deserializes into those records; everything else of the env stays where it is.
struct StateSlot {
    int32_t env;
    int32_t n_ents;         // entities [0, n_ents)
    int32_t cells;          // grid cells [0, cells)
    int32_t scratch_first;  // scratch words [scratch_first, scratch_first + scratch_words)
    int32_t scratch_words;
    int32_t pad;
    int64_t offset;         // of the packed record, in bytes from the start of its chunk's records
};

PG_HD size_t state_ents_off() { return sizeof(EnvHdr) + 2 * sizeof(MT19937); }
PG_HD size_t state_grid_off(const StateSlot &s) { return state_ents_off() + (size_t)s.n_ents * sizeof(Entity); }
PG_HD size_t state_scratch_off(const StateSlot &s) { return state_grid_off(s) + (((size_t)s.cells * sizeof(int16_t) + 15) & ~(size_t)15); }
PG_HD size_t state_record_bytes(const StateSlot &s) {
    return state_scratch_off(s) + (((size_t)s.scratch_words * sizeof(int32_t) + 15) & ~(size_t)15);
}

// s.env's records -> the packed record `rec` (STORE false), or `rec` -> the env's records (STORE true). One warp (one
// thread in the host debug build).
template <bool STORE>
PG_HD void state_move(const KParams &p, const StateSlot &s, unsigned char *rec) {
    static_assert(sizeof(EnvHdr) % 16 == 0 && sizeof(MT19937) % 16 == 0, "16-byte parts");
    const int env = s.env;
    auto vecs = [](void *env_part, unsigned char *rec_part, size_t bytes) {
        if (STORE)
            bank_copy_vecs(env_part, rec_part, (int)bytes);
        else
            bank_copy_vecs(rec_part, env_part, (int)bytes);
    };
    vecs(p.hdr + env, rec, sizeof(EnvHdr));
    vecs(p.rng + env, rec + sizeof(EnvHdr), sizeof(MT19937));
    vecs(p.lvl_rng + env, rec + sizeof(EnvHdr) + sizeof(MT19937), sizeof(MT19937));
    vecs(p.ents + (size_t)env * p.ent_stride, rec + state_ents_off(), (size_t)s.n_ents * sizeof(Entity));
    int16_t *grid = p.grid + (size_t)env * p.grid_stride;
    int16_t *rec_grid = reinterpret_cast<int16_t *>(rec + state_grid_off(s));
    pg_warp_for(s.cells, [=](int k) {
        if (STORE)
            grid[k] = rec_grid[k];
        else
            rec_grid[k] = grid[k];
    });
    int32_t *scratch = p.scratch + (size_t)env * p.scratch_stride + s.scratch_first;
    int32_t *rec_scratch = reinterpret_cast<int32_t *>(rec + state_scratch_off(s));
    pg_warp_for(s.scratch_words, [=](int k) {
        if (STORE)
            scratch[k] = rec_scratch[k];
        else
            rec_scratch[k] = scratch[k];
    });
}

// ---- snapshot slots (pgb200_get_snapshots / pgb200_apply_snapshots): packed records kept in a handle-owned store on
// the device. Every slot has the same size, set by the handle's strides, and holds
//   StateSlot (the record's sizes, as state_slot() makes them) | Entity ghost | the packed record
// The ghost is entity slot ent_cap, where erase_if_needed moves an agent it erases (agent_idx == ent_cap). Nothing in
// a step resets an env on that alone (step_play's done tests the agent against the world's bounds, not its erasure),
// so the code does not rule out such a state between steps, and a snapshot carries the ghost with the record. get_state
// refuses that state instead, since the wire format has no place for the ghost.
struct SnapshotStore {
    unsigned char *slots;     // [count][slot_bytes]; null: the handle has no store
    int64_t slot_bytes;
    int32_t count;            // slots
    int32_t num_envs;
    int32_t games;            // env e plays game e % games of the list
    int32_t pad;
    int32_t *save_from;       // [count] the caller's: env whose state slot s takes at the next apply, -1 = none
    int32_t *load_from;       // [num_envs] the caller's: slot env e takes at the next apply, -1 = none
    int32_t *source;          // [count] env whose state slot s holds, -1 = empty
    const int32_t *persist;   // [games][2] each game's PERSIST_SCRATCH_FIRST and _WORDS
    int32_t *list;            // [num_envs] the envs an apply loaded: game g's at [g, g + 1) * num_envs / games
    unsigned int *counts;     // [games] entries in each game's segment of `list`
};

constexpr size_t kSnapshotGhostOff = sizeof(StateSlot);
constexpr size_t kSnapshotRecordOff = kSnapshotGhostOff + sizeof(Entity);
static_assert(sizeof(StateSlot) % 16 == 0, "16-byte slot parts");

// Slot s takes the current state of env save_from[s], if that is in [0, num_envs): the packed record of the env's live
// part and its ghost entity; then source[s] = env and save_from[s] = -1. One warp (one thread in the host debug build).
PG_HD void snapshot_save(const KParams &p, const SnapshotStore &st, int s) {
    const int env = st.save_from[s];
    if (env < 0 || env >= st.num_envs)
        return;
    const EnvHdr &h = p.hdr[env];
    const int64_t cells = (int64_t)h.main_width * h.main_height;
    StateSlot d{};
    d.env = env;
    d.n_ents = h.n_ents < 0 ? 0 : (h.n_ents < p.ent_stride - 1 ? h.n_ents : p.ent_stride - 1);
    d.cells = cells < 0 ? 0 : (int)(cells < p.grid_stride ? cells : p.grid_stride);
    d.scratch_first = st.persist[2 * (env % st.games)];
    d.scratch_words = st.persist[2 * (env % st.games) + 1];
    unsigned char *slot = st.slots + (size_t)s * (size_t)st.slot_bytes;
    state_move<false>(p, d, slot + kSnapshotRecordOff);
    bank_copy_vecs(slot + kSnapshotGhostOff, p.ents + (size_t)env * p.ent_stride + (p.ent_stride - 1), (int)sizeof(Entity));
    // every lane has read save_from[s] before the warp_for barriers above
    pg_warp_for(1, [=](int) {
        *reinterpret_cast<StateSlot *>(slot) = d;
        st.source[s] = env;
        st.save_from[s] = -1;
    });
}

// Env takes the state slot load_from[env] holds, if the slot is in [0, count), holds a state, and of the env's own game;
// then it is appended to its game's segment of `list` and load_from[env] = -1. An entry refused stays as it is. One
// warp (one thread in the host debug build).
PG_HD void snapshot_load(const KParams &p, const SnapshotStore &st, int env) {
    const int s = st.load_from[env];
    if (s < 0 || s >= st.count)
        return;
    const int src = st.source[s];
    if (src < 0 || src % st.games != env % st.games)
        return;
    unsigned char *slot = st.slots + (size_t)s * (size_t)st.slot_bytes;
    StateSlot d = *reinterpret_cast<const StateSlot *>(slot);
    d.env = env;
    state_move<true>(p, d, slot + kSnapshotRecordOff);
    bank_copy_vecs(p.ents + (size_t)env * p.ent_stride + (p.ent_stride - 1), slot + kSnapshotGhostOff, (int)sizeof(Entity));
    const int g = env % st.games;
    int32_t *const seg = st.list + (size_t)g * (size_t)(st.num_envs / st.games);
    unsigned int *const count = st.counts + g;
    list_append(true, seg, count, env);
    pg_warp_for(1, [=](int) { st.load_from[env] = -1; });
}

#if defined(__CUDACC__)
// Warm the env's working set. A step's logic is one long dependent chain; touched cold, every
// entity record / header line / grid row costs a serial DRAM round trip. Here the 32 lanes issue
// all those line fetches at once (prefetch.global.L2 + L1), so the chain later runs on cache hits.
__device__ __forceinline__ void pg_prefetch_line(const void *ptr) {
    asm volatile("prefetch.global.L1 [%0];" ::"l"(ptr));
}
__device__ __forceinline__ void env_prefetch(const KParams &p, int env) {
    const int lane = (int)(threadIdx.x & 31u);
    const char *hdr = reinterpret_cast<const char *>(p.hdr + env);
    if (lane < (int)((sizeof(EnvHdr) + 127) / 128))
        pg_prefetch_line(hdr + lane * 128);
    const MT19937 *rng = p.rng + env;
    if (lane == 8)
        pg_prefetch_line(&rng->p);
    const Entity *ents = p.ents + (size_t)env * p.ent_stride;
    const int n = p.hdr[env].n_ents;   // first demand load (same line as the prefetch above)
    for (int i = lane; i < n; i += 32) pg_prefetch_line(ents + i);
    // RNG words of the next draw and the grid rows around the agent
    if (lane == 9) {
        int k = rng->p >= 624 ? 0 : rng->p;
        pg_prefetch_line(&rng->mt[k]);
        pg_prefetch_line(&rng->mt[(k + 397) % 624]);
    }
    if (lane >= 16 && lane < 24 && n > 0) {
        const EnvHdr &h = p.hdr[env];
        const Entity &a = ents[h.agent_idx];
        int row = (int)a.y + (lane - 16) - 3;
        if (row >= 0 && row < h.main_height) {
            int col = (int)a.x - 4;
            if (col < 0) col = 0;
            pg_prefetch_line(p.grid + (size_t)env * p.grid_stride + row * h.main_width + col);
        }
    }
    __syncwarp();
}
#endif

// The game steps env plays in one step: repeat[env] with action repeat (REPEAT), at least one, else one
template <bool REPEAT>
PG_HD int env_repeat_count(const KParams &p, int env) {
    if (!REPEAT)
        return 1;
    const int32_t r = p.repeat[env];
    return r > 1 ? r : 1;
}

// Game::step (game.cpp:120-155) up to, not including, the pixel work. One thread.
// LEVEL_CHOICE: the handle has a next_level_seed array. A separate instantiation, so that the logic kernel
// of a handle without one carries no trace of the feature (not even registers held across the step).
// REPEAT: the handle has action repeat: Game::step runs with env's action until a game step resets the env or
// repeat[env] of them have run, and rew is the float sum of their rewards, in order. The sum starts at -0, which
// leaves a single reward's bits as they are. Camera and outputs follow once, for the last game step.
template <class G, class Frame, bool LEVEL_CHOICE = false, bool REPEAT = false>
PG_HD void env_step_logic(const KParams &p, int env) {
#if defined(__CUDA_ARCH__)
    env_prefetch(p, env);
#endif
    Ctx c = make_ctx(p, env);
    const int reps = env_repeat_count<REPEAT>(p, env);
    float rew = -0.f;
    for (int k = 1;; k++) {
        c.h->action = p.action[env];  // vecgame.cpp:388
        bool do_reset;
        if (LEVEL_CHOICE) {
            do_reset = Engine<G>::step_play(c);
            // the caller's choice of the next level is read only by a step that resets, and consumed when that
            // reset takes it
            const int32_t next_seed = do_reset ? p.next_level_seed[env] : -1;
            if (Engine<G>::step_finish(c, do_reset, next_seed))
                p.next_level_seed[env] = -1;
        } else {
            do_reset = Engine<G>::step_play(c);
            Engine<G>::step_finish(c, do_reset, -1);
        }
        if (!REPEAT)
            break;
        rew += c.h->reward;
        if (do_reset || k >= reps)
            break;
    }
    Raster<G, Frame>::prepare_camera(c);
    write_step_outputs(p, env, *c.h);
    if (REPEAT)
        p.rew[env] = rew;
}

// The start of a step on a handle with a pause mask, before anything of the env is touched: records whether env is
// paused in this step and, if it is, writes the outputs a paused step defines (rew = 0, first = 0, and level_end = 0
// with final outputs). Its state, rgb and info slots keep their values. Returns whether env is paused.
template <bool FINAL>
PG_HD bool env_pause_logic(const KParams &p, int env) {
    const uint8_t paused = p.pause[env] != 0;
    p.paused[env] = paused;
    if (paused) {
        p.rew[env] = 0.f;
        p.first[env] = 0;
        if (FINAL)
            p.level_end[env] = 0;
    }
    return paused != 0;
}

// Phase A of a step with final outputs: Game::step up to the reset decision, with the cause of a level end
// in level_end[env]. An env that does not reset finishes as in env_step_logic. One that does gets the camera
// of its final state, and the rest of its step (the reset and the scalar outputs) waits for phase B,
// env_finish_logic. Returns whether the env resets.
// REPEAT: the game steps of env_step_logic<REPEAT> that do not reset run here; level_end is the last one's. rew gets
// the sum of their rewards, to which phase B adds the reward of a game step that resets.
template <class G, class Frame, bool REPEAT = false>
PG_HD bool env_step_logic_final(const KParams &p, int env) {
#if defined(__CUDA_ARCH__)
    env_prefetch(p, env);
#endif
    Ctx c = make_ctx(p, env);
    const int reps = env_repeat_count<REPEAT>(p, env);
    float rew = -0.f;
    bool do_reset;
    for (int k = 1;; k++) {
        c.h->action = p.action[env];  // vecgame.cpp:388
        uint8_t cause = 0;
        do_reset = Engine<G>::template step_play<true>(c, &cause);
        p.level_end[env] = cause;
        if (do_reset)
            break;
        Engine<G>::step_finish(c, false, -1);
        if (!REPEAT)
            break;
        rew += c.h->reward;
        if (k >= reps)
            break;
    }
    Raster<G, Frame>::prepare_camera(c);
    if (!do_reset)
        write_step_outputs(p, env, *c.h);
    if (REPEAT)
        p.rew[env] = rew;
    return do_reset;
}

// One env of the logic kernel: INIT the first reset, otherwise a step. PAUSE: unless the pause mask holds env still.
// FINAL: phase A of a two-phase step, which appends env to p.reset_list when its level ends. LEVEL_CHOICE: see
// env_step_logic (a two-phase step's resets take the caller's choice in phase B). REPEAT: action repeat (see
// env_step_logic); a paused env plays no game step.
template <class G, class Frame, bool INIT, bool LEVEL_CHOICE, bool FINAL, bool PAUSE, bool REPEAT = false>
PG_HD void env_logic(const KParams &p, int env) {
    static_assert(!(LEVEL_CHOICE && FINAL), "phase A never resets");
    static_assert(!(INIT && REPEAT), "the initial reset plays no game step");
    if (INIT)
        env_init_logic<G, Frame>(p, env);
    else if (PAUSE && env_pause_logic<FINAL>(p, env)) {
    } else if (FINAL) {
        list_append(env_step_logic_final<G, Frame, REPEAT>(p, env), p.reset_list, p.reset_count, env);
    } else
        env_step_logic<G, Frame, LEVEL_CHOICE, REPEAT>(p, env);
}

// Where a lookahead handle's reset takes its level from: the bank where it holds the seed (BANK), else the env's
// lookahead slot where it holds the seed for options like the env's, else generation. Counts the choice in
// p.look.served.
template <class G, bool BANK>
struct LookaheadSource {
    const KParams &p;
    int env;
    PG_HD bool copy_level(Ctx &c) const {
        int from = 2;
        if (BANK && bank_copy_level<G>(c, p.bank)) {
            from = 1;
        } else {
            unsigned char *slot = lookahead_slot(p.look, env);
            if (slot_key(slot) == c.h->current_level_seed && slot_usable(slot) != 0 && bank_options_match(c.h->options, p.look.slot.options)) {
                bank_copy_slot<G>(c, slot, p.look.slot);
                from = 0;
            }
        }
#if defined(__CUDA_ARCH__)
        if ((threadIdx.x & 31u) == 0)
            atomicAdd(p.look.served + from, 1ull);
#else
        p.look.served[from]++;
#endif
        return from != 2;
    }
};

// The level env's next reset is predicted to play: its current level again while episodes_remaining != 0, otherwise
// the next draw of level_seed_rand_gen (a completed level of use_sequential_levels goes on by +997 instead, and
// misses). Unless the bank holds it (`bank`) or the env's slot already does, the slot is keyed with the prediction,
// marked not usable, and env is appended to p.look.list for the lookahead kernel. An env whose generator an older blob
// left half-twisted, or whose options are not the handle's, keeps its slot as it is.
PG_HD void lookahead_predict(const KParams &p, int env, bool bank) {
    const EnvHdr &h = p.hdr[env];
    int32_t seed = h.current_level_seed;
    if (h.episodes_remaining == 0 && !rand_peek_randint(p.lvl_rng[env], h.level_seed_low, h.level_seed_high, &seed))
        return;
    if (!bank_options_match(h.options, p.look.slot.options))
        return;
    if (bank && bank_find(p.bank.seeds, *p.bank.count, seed) >= 0)
        return;
    unsigned char *slot = lookahead_slot(p.look, env);
    if (slot_key(slot) == seed)
        return;
    // lane 0 keys the slot once every lane has read the old key
#if defined(__CUDA_ARCH__)
    __syncwarp();
    if ((threadIdx.x & 31u) == 0)
#endif
    {
        slot_key(slot) = seed;
        slot_usable(slot) = 0;
    }
    list_append(true, p.look.list, p.look.count, env);
#if defined(__CUDA_ARCH__)
    __syncwarp();
#endif
}

// Phase B: the rest of Game::step for an env whose level ended in phase A. The reset reads and consumes the
// env's next_level_seed entry as env_step_logic<LEVEL_CHOICE> does; then Game::observe's camera and scalars.
// BANK: the handle has a level bank, which the reset copies the level from when it holds it.
// LOOK: the handle has level lookahead: the reset's level comes from LookaheadSource, and the env's next one is
// predicted (lookahead_predict).
// REPEAT: the handle has action repeat; rew then adds the reward after the reset to phase A's sum in rew.
template <class G, class Frame, bool BANK = false, bool LOOK = false, bool REPEAT = false>
PG_HD void env_finish_logic(const KParams &p, int env) {
    const float rew = REPEAT ? p.rew[env] : 0.f;
    Ctx c = make_ctx(p, env);
    const int32_t next_seed = p.next_level_seed ? p.next_level_seed[env] : -1;
    if constexpr (LOOK) {
        const LookaheadSource<G, BANK> src{p, env};
        if (Engine<G>::template step_finish<BANK, const LookaheadSource<G, BANK>>(c, true, next_seed, &p.bank, &src))
            p.next_level_seed[env] = -1;
        lookahead_predict(p, env, BANK);
    } else {
        if (Engine<G>::template step_finish<BANK>(c, true, next_seed, &p.bank))
            p.next_level_seed[env] = -1;
    }
    Raster<G, Frame>::prepare_camera(c);
    write_step_outputs(p, env, *c.h);
    if (REPEAT)
        p.rew[env] = rew + c.h->reward;
}

// Level bank build: per-warp staging, the env's own record at the handle's capacities (EnvHdr, entities, grid,
// rand_gen, level-generation scratch), 16-byte aligned parts
PG_HD size_t bank_stage_bytes(const KParams &p) {
    return sizeof(EnvHdr) + (size_t)p.ent_stride * sizeof(Entity) + (((size_t)p.grid_stride * sizeof(int16_t) + 15) & ~(size_t)15) +
           sizeof(MT19937) + (((size_t)p.scratch_stride * sizeof(int32_t) + 15) & ~(size_t)15);
}

// Generates the level of `seed` of the launch's game in `stage`, as a reset would from the state init_constants
// leaves with the handle's options, then stores it in the slot slot_of() returns (laid out as `b` describes), marked
// usable if it fits the game's slot. One warp (or one thread in the host debug build).
template <class G, class SlotOf>
PG_HD void bank_generate_level(const KParams &p, const LevelBank &b, int32_t seed, SlotOf slot_of, unsigned char *stage) {
    Ctx c;
    c.h = reinterpret_cast<EnvHdr *>(stage);
    c.ents = reinterpret_cast<Entity *>(stage + sizeof(EnvHdr));
    c.grid = reinterpret_cast<int16_t *>(stage + sizeof(EnvHdr) + (size_t)p.ent_stride * sizeof(Entity));
    c.rng = reinterpret_cast<MT19937 *>(reinterpret_cast<unsigned char *>(c.grid) + (((size_t)p.grid_stride * sizeof(int16_t) + 15) & ~(size_t)15));
    c.scratch = reinterpret_cast<int32_t *>(c.rng + 1);
    c.lvl_rng = nullptr;  // game_reset never draws a level seed
    c.assets = p.assets;
    c.ent_cap = p.ent_stride - 1;
    c.grid_cap = p.grid_stride;
    c.scratch_cap = p.scratch_stride;
    c.obst_hi = -1;
    c.rot_scratch_raw = nullptr;
    c.blit_list = nullptr;
    c.cell_spill = nullptr;
    G::init_constants(c);
    EnvHdr &h = *c.h;
    h.options = p.options;
    h.options.center_agent = BANK_CENTER_AGENT_UNSET;
    h.game_id = p.game_id;
    h.fixed_asset_seed = p.fixed_asset_seed;
    h.level_seed_low = p.level_seed_low;
    h.level_seed_high = p.level_seed_high;
    h.current_level_seed = seed;
    h.episodes_remaining = 1;
    ctx_refresh(c);
    mt_seed(*c.rng, (uint32_t)h.current_level_seed);
    G::game_reset(c);
    unsigned char *slot = slot_of();
    const bool usable = h.max_ents_seen <= G::ENT_CAP && h.grid_size <= G::GRID_CAP && h.agent_idx < c.ent_cap;
    if (usable) {
        bank_copy_vecs(slot + BANK_SLOT_HEAD, &h, (int)sizeof(EnvHdr));
        bank_copy_vecs(slot + b.ents_off, c.ents, h.n_ents * (int)sizeof(Entity));
        int16_t *dg = reinterpret_cast<int16_t *>(slot + b.grid_off);
        const int16_t *sg = c.grid;
        pg_warp_for(h.grid_size, [=](int k) { dg[k] = sg[k]; });
        bank_copy_vecs(slot + b.rng_off, c.rng, (int)sizeof(MT19937));
        int32_t *ds = reinterpret_cast<int32_t *>(slot + b.scratch_off);
        const int32_t *ss = c.scratch + G::PERSIST_SCRATCH_FIRST;
        pg_warp_for(G::PERSIST_SCRATCH_WORDS, [=](int k) { ds[k] = ss[k]; });
    }
    *reinterpret_cast<int32_t *>(slot) = usable ? 1 : 0;  // every lane stores the same value
}

// The level p.look.list[item]'s slot is keyed with, generated into the slot (lookahead kernel, bulk fill)
template <class G>
PG_HD void lookahead_generate(const KParams &p, int item, unsigned char *stage) {
    unsigned char *slot = lookahead_slot(p.look, p.look.list[item]);
    bank_generate_level<G>(p, p.look.slot, slot_key(slot), [=] { return slot; }, stage);
}

// Profiling variant (-DPG_PHASE_TIMING): the setup kernel's phases, SM cycles of env's last frame in header slots
// the render kernel does not write (it takes 0, 5, 6, 7): 1 setup_frame, 2 entity blits (with the tiles and
// rotated sprites they reserved, and the overlays), 3 frame_build, 4 frame_tile_alloc, 8 frame_cells_finish,
// 9 the store of the record. A reset earlier in the same step leaves level-generation cycles in these slots;
// the setup kernel overwrites them.
#if defined(PG_PHASE_TIMING) && defined(__CUDA_ARCH__)
#define PG_SETUP_PHASE_BEGIN long long _pg_s0 = clock64()
#define PG_SETUP_PHASE(id)                                    \
    do {                                                      \
        const long long _pg_s1 = clock64();                   \
        if (lane == 0)                                        \
            p.hdr[env].dbg_phase[id] = (uint32_t)(_pg_s1 - _pg_s0); \
        _pg_s0 = _pg_s1;                                      \
    } while (0)
#else
#define PG_SETUP_PHASE_BEGIN do { } while (0)
#define PG_SETUP_PHASE(id) do { } while (0)
#endif

// ---- setup kernel body: one warp (lanes `lane` of `nlanes`) prepares everything about env's frame that
// does not depend on pixels or cells: camera, spans, background / overlay / entity blits. `f` is the warp's
// own record (shared memory on the device), which holds whatever the warp's previous env left in it: every
// field is written for this frame before it is read.
template <class G, class Setup>
PG_HD void env_setup_frame(const KParams &p, int env, Setup &f, int lane, int nlanes) {
    PG_SETUP_PHASE_BEGIN;
    Ctx c = make_ctx(p, env);
    using R = Raster<G, Setup>;
    R::setup_frame(c, f, p.snap != 0, lane, nlanes);
#if defined(__CUDA_ARCH__)
    __syncwarp();
#endif
    PG_SETUP_PHASE(1);
    R::build_entity_blits(c, f, lane, nlanes);
#if defined(__CUDA_ARCH__)
    __syncwarp();
#endif
    if (f.n_jobs > 0) {
        R::frame_tiles(c, f, lane, nlanes);
#if defined(__CUDA_ARCH__)
        __syncwarp();
#endif
    }
    if (G::DEFER_ROTATED) {
        R::frame_rots(c, f, lane, nlanes);
#if defined(__CUDA_ARCH__)
        __syncwarp();
#endif
    }
    if (lane == 0)
        R::frame_append_overlays(f);
    // cells: pixel -> cell lookups, classification, the tiles they need and where those will sit in the
    // render CTA's arena
    if (G::DRAWS_GRID) {
#if defined(__CUDA_ARCH__)
        __syncwarp();
#endif
        PG_SETUP_PHASE(2);
        R::frame_build(c, f, lane, nlanes, 0);
#if defined(__CUDA_ARCH__)
        __syncwarp();
#endif
        PG_SETUP_PHASE(3);
        R::frame_tile_alloc(c, f, p.tiles, lane, nlanes);
#if defined(__CUDA_ARCH__)
        __syncwarp();
#endif
        PG_SETUP_PHASE(4);
        R::frame_cells_finish(c, f, lane, nlanes);
        PG_SETUP_PHASE(8);
    } else {
        PG_SETUP_PHASE(2);
        R::frame_build(c, f, lane, nlanes, 0);  // background row offsets only
        PG_SETUP_PHASE(3);
        PG_SETUP_PHASE(4);
        PG_SETUP_PHASE(8);
    }
}

// The setup kernel's result, the FrameSharedT prefix of the warp's record `f`, stored to env's slot of
// p.frame_setup with 16-byte vectors, the warp's lanes side by side (one lane in the host debug build). The render
// kernel stages it from there. The rest of the record is the setup kernel's own scratch and stays where it is.
template <class Setup>
PG_HD void env_store_frame(const KParams &p, int env, const Setup &f) {
    using Shared = typename Setup::Shared;
    static_assert(sizeof(Shared) % 16 == 0, "the record is stored in 16-byte vectors");
    bank_copy_vecs(p.frame_setup + (size_t)env * p.frame_setup_stride, static_cast<const Shared *>(&f), (int)sizeof(Shared));
}

// Host debug harness twin of the bulk copies that stage the frame's tiles
template <class Frame>
PG_HD void env_stage_tiles_serial(const KParams &p, Frame &f) {
    const int nj = f.n_tjobs < MAX_TILE_JOBS ? f.n_tjobs : MAX_TILE_JOBS;
    for (int j = 0; j < nj; j++)
        for (int w = 0; w < (int)f.tjob_words[j]; w++) f.arena[f.tjob_dst[j] + w] = p.tiles.texels[f.tjob_src[j] + w];
}

// Compose the rows row_first, row_first + row_step, ... of the frame (`lane` of `nlanes` threads own them)
template <class G, class Frame>
PG_HD void env_render_compose(const KParams &p, Frame &f, int row_first, int row_step, int lane, int nlanes) {
    Raster<G, Frame>::compose_rows(f, f.fb, row_first, row_step, lane, nlanes, p.atlas);
}

// Fill one tile of the global table (TileTable): tile (slot, tw, th) = the texels an un-clipped
// drawImage of the sprite at snapped size tw x th samples, by the general path's own arithmetic.
PG_HD void tile_table_fill(const SpriteDesc *sprites, const uint32_t *index, uint32_t *texels, const uint32_t *atlas, int slot, int tw, int th, int tid,
                           int nthreads) {
    Blit b;
    make_image_blit(b, 0.0, 0.0, (double)tw, (double)th, sprites[slot], false, 256, true);
    uint32_t *dst = texels + index[(slot * MAX_TILE_DIM + (tw - 1)) * MAX_TILE_DIM + (th - 1)];
    const int words = tile_words(tw, th);
    for (int i = tid; i < words; i += nthreads) {
        const int dy = i / tw, dx = i - dy * tw;
        dst[i] = dy < th ? tile_texel(b, atlas, dx, dy) : 0u;
    }
}

// Frame sizing per game: visible window (cells per side) and entity capacity.
// VIEW = cells per side of the largest visible grid window: G::MAX_VIEW_CELLS for the game's usual view,
// G::FULL_VIEW_CELLS for the whole-world view the scrolling games draw with center_agent = false
template <class G, int VIEW = G::MAX_VIEW_CELLS>
struct FrameFor {
    using type = FrameT<(G::DRAWS_GRID ? VIEW : 1), G::MAX_VISIBLE_ENTS, G::MAX_ROT_BLITS>;
    using setup = FrameSetupT<(G::DRAWS_GRID ? VIEW : 1), G::MAX_VISIBLE_ENTS, G::MAX_ROT_BLITS>;
    using shared = typename type::Shared;
};

}  // namespace pg
