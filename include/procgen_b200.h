/* procgen_b200 — C ABI of the H100 (sm_90a) vectorised Procgen backend (libprocgen_b200.so).
 *
 * Part 1 is the libenv interface that the reference's libenv.so exports and that gym3's
 * `CEnv` binds through cffi (reference: procgen/src/vecgame.cpp:42-99 for the seven libenv_*
 * entry points, :437-457 for get_state/set_state, declared to cffi at procgen/env.py:132-135).
 * The struct layouts restate gym3==0.3.3 `gym3/libenv.h` (pinned by environment.yml:12), which is
 * not vendored in the reference tree; they are reconstructed from their uses in vecgame.cpp:212-282
 * (libenv_tensortype), vecoptions.cpp:4-54 (libenv_option[s]) and vecgame.cpp:30-40,74-83
 * (libenv_buffers: bufs[space_idx * num_envs + env_idx]).
 *
 * Part 2 is the device-resident extension: the same environment, but observations, rewards,
 * firsts, infos and actions stay in HBM and are exposed as raw device pointers (plain pointers
 * and sizes, no framework types) so a caller can wrap them as tensors without a host round trip.
 */
#ifndef PROCGEN_B200_H
#define PROCGEN_B200_H

#include <stdbool.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#if defined(_WIN32)
#define LIBENV_API __declspec(dllexport)
#else
#define LIBENV_API __attribute__((visibility("default")))
#endif

/* ------------------------------------------------------------------ Part 1: libenv */

#define LIBENV_VERSION 1
#define LIBENV_MAX_NAME_LEN 128
#define LIBENV_MAX_NDIM 16

enum libenv_dtype {
    LIBENV_DTYPE_UNUSED = 0,
    LIBENV_DTYPE_UINT8 = 1,
    LIBENV_DTYPE_INT32 = 2,
    LIBENV_DTYPE_FLOAT32 = 3,
};

enum libenv_scalar_type {
    LIBENV_SCALAR_TYPE_UNUSED = 0,
    LIBENV_SCALAR_TYPE_REAL = 1,
    LIBENV_SCALAR_TYPE_DISCRETE = 2,
};

enum libenv_space_name {
    LIBENV_SPACE_UNUSED = 0,
    LIBENV_SPACE_OBSERVATION = 1,
    LIBENV_SPACE_ACTION = 2,
    LIBENV_SPACE_INFO = 3,
};

union libenv_value {
    uint8_t uint8;
    int32_t int32;
    float float32;
};

struct libenv_tensortype {
    char name[LIBENV_MAX_NAME_LEN];
    enum libenv_scalar_type scalar_type;
    enum libenv_dtype dtype;
    int shape[LIBENV_MAX_NDIM];
    int ndim;
    union libenv_value low;
    union libenv_value high;
};

struct libenv_option {
    char name[LIBENV_MAX_NAME_LEN];
    enum libenv_dtype dtype;
    int count;
    void *data;
};

struct libenv_options {
    struct libenv_option *items;
    int count;
};

struct libenv_buffers {
    void **ob;      /* [n_ob_spaces * num_envs], index space_idx * num_envs + env_idx */
    float *rew;     /* [num_envs] */
    uint8_t *first; /* [num_envs] */
    void **info;    /* [n_info_spaces * num_envs] */
    void **ac;      /* [n_ac_spaces * num_envs] */
};

typedef void libenv_env;

/* vecgame.cpp:43-45 */
LIBENV_API int libenv_version(void);

/* vecgame.cpp:47-50. Options consumed: every option of VecGame::VecGame (vecgame.cpp:183-190:
 * env_name, num_levels, start_level, num_actions, rand_seed, num_threads, resource_root,
 * render_human) and of Game::parse_options (game.cpp:42-75).  Unknown options are fatal
 * (vecoptions.cpp:34-38).  num_threads is accepted and ignored: stepping is one asynchronous
 * kernel launch per act().  resource_root names the directory holding assets.pack (or the pack
 * file itself).  Extra, optional int32 options understood by this backend only:
 *   cuda_device        device ordinal (default: current device)
 *   env_index_offset   global index of env 0 when one logical VecGame of `env_index_total` envs
 *   env_index_total    is sharded over several handles/GPUs; the per-env seed chain
 *                      (vecgame.cpp:301-314) and game_n are replayed for the global indices
 *   snap_target_rect   uint8 bool, default 1: Qt>=6 integer snapping of un-rotated image targets */
LIBENV_API libenv_env *libenv_make(int num_envs, const struct libenv_options options);

/* vecgame.cpp:52-72; `types` may be NULL to query the count. */
LIBENV_API int libenv_get_tensortypes(libenv_env *handle, enum libenv_space_name name, struct libenv_tensortype *types);

/* vecgame.cpp:74-83 -> VecGame::set_buffers (:333-361): stores the caller-owned HOST pointers and
 * performs the initial reset + observe of every env. */
LIBENV_API void libenv_set_buffers(libenv_env *handle, struct libenv_buffers *bufs);

/* vecgame.cpp:85-88 -> VecGame::observe (:363-376): waits for the step in flight and fills the
 * host buffers given to libenv_set_buffers. */
LIBENV_API void libenv_observe(libenv_env *handle);

/* vecgame.cpp:90-93 -> VecGame::act (:378-401): copies the actions out of the host buffers
 * (they are only valid during this call) and starts the step asynchronously. */
LIBENV_API void libenv_act(libenv_env *handle);

/* vecgame.cpp:95-98 */
LIBENV_API void libenv_close(libenv_env *handle);

/* State snapshots — replaces get_state / set_state, src/vecgame.cpp:437-457 (declared to cffi at
 * procgen/env.py:132-135). The blob is the reference's own wire format, byte for byte
 * (Game::serialize game.cpp:170-229, BasicAbstractGame::serialize basic-abstract-game.cpp:1169-1223,
 * Entity::serialize entity.cpp:90-131, RandGen::serialize randgen.cpp:100-107, per-game tails): a
 * state saved by the reference loads here and vice versa. get_state returns the number of bytes
 * written (a too small buffer is fatal, like the reference's fassert); set_state also re-renders
 * the env's observation and rewrites its rew / first / info slots from the restored state (Game::observe).
 * Both wait for the step in flight. They are the one-env case of pgb200_get_states / pgb200_set_states (Part 2);
 * a malformed blob is fatal with `fatal: set_state: <check> (env <index>)`. */
LIBENV_API int get_state(libenv_env *handle, int env_idx, char *data, int length);
LIBENV_API void set_state(libenv_env *handle, int env_idx, char *data, int length);

/* ------------------------------------------------------------------ Part 2: device-resident */

struct pgb200_device_buffers {
    uint8_t *rgb;                  /* [num_envs][64][64][3] uint8, device */
    float *rew;                    /* [num_envs] */
    uint8_t *first;                /* [num_envs] */
    int32_t *prev_level_seed;      /* [num_envs] info */
    uint8_t *prev_level_complete;  /* [num_envs] info */
    int32_t *level_seed;           /* [num_envs] info */
    int32_t *action;               /* [num_envs], written by the caller before pgb200_act_device */
    int32_t num_envs;
    int32_t device;                /* CUDA device ordinal, -1 for the CPU debug build */
    void *stream;                  /* cudaStream_t all work of this handle is ordered on */
};

/* Returns 0 on success. The first call performs the initial reset + render (the work
 * libenv_set_buffers does in host mode). Pointers stay valid until libenv_close. */
LIBENV_API int pgb200_get_device_buffers(libenv_env *handle, struct pgb200_device_buffers *out);

/* Per-env level choice: `*out` = this handle's int32 array next_level_seed[num_envs] (device memory;
 * host memory in the CPU debug build), allocated and filled with -1 by the first call, which also
 * performs the initial reset if it has not happened yet. The pointer stays valid until libenv_close.
 * At every reset inside a step (an episode end, the timeout, or action -1), env e reads
 * s = next_level_seed[e]: s >= 0 makes the new level's seed s instead of a draw from the env's
 * level_seed_rand_gen (not advanced) or the +997 of use_sequential_levels (later levels continue from
 * s + 997), and the step writes -1 back (the override is consumed); s < 0 leaves the reset as it is. Any
 * s in [0, 2^31) is accepted, also outside [start_level, start_level + num_levels). Indices are the
 * handle's own (env n of a joint list plays game n % G; local indices of a shard). The initial reset
 * is not affected; to start envs on chosen levels, write overrides and step once with action -1.
 * get_state / set_state neither read nor write the array (pending overrides survive set_state).
 * Ordering: with pgb200_act_device, write the array on the handle's stream before the call, like the
 * action buffer; with libenv_act, the writes must be complete before the call. Returns 0. */
LIBENV_API int pgb200_get_next_level_seeds(libenv_env *handle, int32_t **out);

/* Final outputs: the frame each env's level ended in, and why it ended. A step that ends an episode resets
 * the env inside it and returns the next level's first frame (Game::step, game.cpp:120-155); these arrays
 * keep what that reset hides, e.g. the state V(s_T) of a truncated episode is computed on.
 *   rgb        [num_envs][64][64][3] uint8
 *   level_end  [num_envs] uint8
 * Device memory (host memory in the CPU debug build), also for a handle with host buffers: there the arrays
 * are complete once libenv_observe returns. The first call allocates them, zero-filled, performs the
 * initial reset if it has not happened yet and returns 0; from then on every step of the handle fills them
 * (there is no off switch). The pointers stay valid until libenv_close.
 * After every step, level_end[e] says whether env e's level was reset inside that step, and why, in the
 * order the reference tests it (game.cpp:132-134):
 *   0                          no reset; rgb[e] is left as it was
 *   PGB200_LEVEL_END_GAME      the game ended the level: the agent died or completed it (prev_level_complete
 *                              tells which)
 *   PGB200_LEVEL_END_TIMEOUT   the game did not, but the episode reached its step limit (a truncation)
 *   PGB200_LEVEL_END_CALLER    neither: the reset came from action -1
 * and where it is not 0, rgb[e] is the frame Game::observe would have rendered had the step not reset.
 * level_end[e] != 0 exactly where first[e] == 1, with one exception: under use_sequential_levels a
 * completed level resets with first = 0 (game.cpp:148-150) and reports PGB200_LEVEL_END_GAME.
 * Every other output of the step (rgb, rew, first, the infos, the consumer output, next_level_seed
 * consumption, the state) is what it is without this call. The initial reset, get_state and set_state
 * neither read nor write the arrays. CUDA graphs: the first call is refused (-1) while the handle's stream
 * captures; a captured step keeps whether final outputs were on at capture.
 * pgb200_kernel_timing_begin returns -1 on a handle with final outputs. */
#define PGB200_LEVEL_END_GAME 1
#define PGB200_LEVEL_END_TIMEOUT 2
#define PGB200_LEVEL_END_CALLER 3
struct pgb200_final_outputs {
    uint8_t *rgb;        /* [num_envs][64][64][3] */
    uint8_t *level_end;  /* [num_envs] */
};
LIBENV_API int pgb200_get_final_outputs(libenv_env *handle, struct pgb200_final_outputs *out);

/* Per-env pause: `*out` = this handle's uint8 array pause[num_envs] (device memory; host memory in the CPU
 * debug build), allocated and filled with 0 by the first call, which also performs the initial reset if it has
 * not happened yet. Returns 0. The pointer stays valid until libenv_close. A step does not consume an entry:
 * it stays in force until the caller clears it. In every step, an env e with pause[e] != 0 is paused:
 *   - its state is untouched, byte for byte (both RNGs, cur_time: a paused step does not count toward the time
 *     limit, the entities, the grid), and its action, -1 included, is ignored;
 *   - its next_level_seed entry is neither read nor consumed;
 *   - rgb[e] and the three info slots keep their values; rew[e] = 0 and first[e] = 0, so that sums of rew and
 *     counts of first over all envs stay correct;
 *   - with final outputs, level_end[e] = 0 and the final rgb[e] keeps its value;
 *   - with the consumer output, the ring moves on for every env (one ring position per handle): a paused env's
 *     newest slot gets its current frame again, so its k-frame stack repeats the frame it is paused on (the older
 *     frames are not zeroed: first = 0).
 * Every env that is not paused steps exactly as on a handle without the mask, and an all-zero mask gives the
 * outputs and states of a handle that never called this. Only the first kernel of a step reads the mask, so
 * rewriting it while a step runs cannot split one env's step. Indices are the handle's own (env n of a joint
 * list plays game n % G; local indices of a shard). get_state / set_state neither read nor write the mask;
 * set_state into a paused env works as always, and the env stays paused.
 * Ordering as for next_level_seed: with pgb200_act_device, write the mask on the handle's stream before the
 * call; with libenv_act, the writes must be complete before the call. CUDA graphs: the first call is refused
 * (-1) while the handle's stream captures; a captured step reads the mask only if it existed at capture, and
 * then reads its contents at every replay. A handle without the mask runs the kernels it ran before. */
LIBENV_API int pgb200_get_pause_mask(libenv_env *handle, uint8_t **out);

/* Action repeat (frame skip): `*out` = this handle's int32 array repeat[num_envs] (device memory; host memory in
 * the CPU debug build), allocated with every entry 1 by the first call, which also performs the initial reset if
 * it has not happened yet. Returns 0. The pointer stays valid until libenv_close. A step reads the array and
 * never changes it. In every step, an env e with repeat[e] = r:
 *   - plays max(r, 1) game steps (Game::step) with its action, and stops after the first whose level ends (game
 *     end, time limit, action -1, or a completed level with use_sequential_levels). Action -1 thus plays one, and
 *     the time limit bounds the game steps of any r;
 *   - reports rew[e] = the float sum of those game steps' rewards, in order; first[e], the three info slots and,
 *     with final outputs, level_end[e] are the last game step's, and rgb[e] is the frame of the final state. The
 *     final rgb[e] of final outputs is the frame of the state the level ended in;
 *   - takes its next_level_seed entry at the one reset the step can contain, as without action repeat.
 * A paused env (pgb200_get_pause_mask) plays no game step, whatever its entry. The rollout and the consumer ring
 * move on once per step. get_state / set_state, snapshots, the level bank and level lookahead neither read nor
 * write the array. An all-ones array gives the outputs and states of a handle that never called this, which runs
 * the kernels it ran before. Ordering and CUDA graphs as for the pause mask: the first call is refused (-1) while
 * the handle's stream captures, and a captured step reads the array only if it existed at capture, then reads its
 * contents at every replay. */
LIBENV_API int pgb200_get_action_repeat(libenv_env *handle, int32_t **out);

/* Level bank: levels generated once and copied in at reset. A generated level is a pure function of the game, the
 * options and the seed, so a handle that keeps resetting onto the same few hundred seeds (num_levels = 200 or
 * 500, a held-out seed list, a level-replay buffer) can keep them instead of generating them again.
 * pgb200_build_level_bank banks `seeds[0, count)` (host memory; every seed in [0, 2^31); duplicates are allowed)
 * for every game of the handle's list. The first call allocates room for max(count, capacity) distinct seeds per
 * game; that capacity is then fixed. A later call rebuilds the bank in place, on the handle's stream and ordered
 * with its steps, so graphs captured earlier stay valid and see the new bank. count == 0 empties it. Performs the
 * initial reset if it has not happened yet, and returns when the bank is built. Returns 0, or -1 (nothing changed)
 * when a seed is out of range, there are more distinct seeds than the capacity, a first call has
 * max(count, capacity) == 0 (a bank that could never hold a level), or the handle's stream is capturing (the call
 * allocates and waits). Slots are sized per game of the list; a level that needs more entities or cells than its
 * game's capacities (possible only in a joint list) is generated at every reset instead.
 * At every reset inside a step, the new level's seed s is chosen as always (game end, time limit, action -1, a
 * next_level_seed override, the +997 of sequential levels). If s is banked and the env's options are the ones the
 * bank was generated with (all but center_agent, which level generation only writes; an env can differ only
 * after set_state of a blob made under other options), the reset copies the banked level instead of generating
 * it. Every output and every state byte is identical to a handle without a bank: its only effect is speed.
 * The initial reset, get_state / set_state, the wire format and next_level_seed consumption are unaffected; a
 * paused env never resets; phase B of final outputs uses the bank like any other reset.
 * CUDA graphs: a captured step uses the bank if one existed at capture, and a rebuild is seen by later replays;
 * a step captured without a bank never uses one. A handle without a bank runs the kernels it ran before.
 * pgb200_level_bank_info: *levels = the distinct seeds banked now, *bytes = the device memory the bank holds
 * (0 and 0 without one). Returns 0. */
LIBENV_API int pgb200_build_level_bank(libenv_env *handle, const int32_t *seeds, int count, int capacity);
LIBENV_API int pgb200_level_bank_info(libenv_env *handle, int *levels, int64_t *bytes);

/* Level lookahead: each env's next level generated while its current episode plays. With num_levels = 0 (the
 * unbounded level distribution) no bank can hold the levels, and an episode end generates its next level inside the
 * step, on one warp, which sets the step's time for caveflyer, jumper and leaper. An env's next seed is known as
 * soon as its episode starts (the next draw of its level seed generator), so a lookahead handle generates that
 * level into a slot of its own beside the frames of the step, and the reset at the episode's end copies it.
 * pgb200_enable_level_lookahead performs the initial reset if it has not happened yet, gives every env a slot sized
 * by its own game (in the bank's slot layout: 24-77 KB, so about 5 GB for coinrun at 65 536 envs), generates each
 * env's predicted next level into it and returns. A second call does nothing and returns 0; -1 (nothing changed)
 * while the handle's stream is capturing. There is no off switch; the memory is released by libenv_close.
 * At every reset inside a step the seed is chosen as always (game end, time limit, action -1, a next_level_seed
 * override, the +997 of sequential levels). A bank that holds it serves the level; otherwise the env's slot does if
 * it holds that seed for the env's options; otherwise the level is generated. Every output and every state byte,
 * error bits and max_ents_seen included, is the one a handle without lookahead gives: its only effect is speed.
 * After each such reset the env's next seed is predicted (its current seed while episodes_remaining != 0, else the
 * next draw of its level seed generator) and generated into its slot unless a bank or the slot already holds it.
 * A prediction can miss: an override, set_state, or a completed level of use_sequential_levels (+997; the draw is
 * predicted) lead to a reset that generates. The initial reset, get_state / set_state, the wire format, override
 * consumption, paused envs, final outputs, the consumer output and the bank are unaffected.
 * CUDA graphs: a step captured after the call uses lookahead at every replay, one captured before it never does. A
 * handle without lookahead runs the kernels it ran before.
 * pgb200_level_lookahead_info: out[0] resets served from a lookahead slot, out[1] resets served from the bank,
 * out[2] resets that generated (all three counted from the call on), out[3] the device bytes lookahead holds (slots
 * and staging); all 0 without lookahead. Returns 0, or -1 while the handle's stream is capturing. */
LIBENV_API int pgb200_enable_level_lookahead(libenv_env *handle);
LIBENV_API int pgb200_level_lookahead_info(libenv_env *handle, int64_t *out /* [4] */);

/* Rollout: every step also stores its rgb, rew and first into a ring of `slots` slots, so that a learner's rollout
 * storage is filled by the render kernel itself instead of by a copy of the outputs after each step (the next step
 * overwrites them). The arrays are slot-major, so rgb + t * num_envs * 12288 is one contiguous [num_envs][64][64][3]
 * block, the shape of a learner's obs_buf[t]:
 *   rgb    [slots][num_envs][64][64][3]  uint8
 *   rew    [slots][num_envs]             float
 *   first  [slots][num_envs]             uint8
 *   cursor [1]                           int32, the slot the latest step (or the first call) wrote
 * They are handle-owned device memory (host memory in the CPU debug build), valid until libenv_close, which frees
 * them; there is no off switch. The first call performs the initial reset if it has not happened yet, allocates the
 * arrays, writes the current rgb, rew and first into slot 0, sets *cursor = 0, waits and returns 0. A later call with
 * the same `slots` returns the same pointers. Returns -1 (nothing changed) when slots < 2, when the ring's byte size
 * overflows, when a later call asks for a different `slots`, or for the first call while the handle's stream is
 * capturing.
 * The invariant: after every step, *cursor has moved from c to c' = (c + 1) % slots and slot c' holds exactly that
 * step's rgb, rew and first, byte for byte. Nothing else any step outputs changes. So with final outputs the slot
 * holds the first frame of the next level (what rgb holds), not the final frame; a paused env's slot holds the frame
 * it is paused on with rew = 0 and first = 0. Every launch shape, joint game list and view, and host-buffer handles
 * follow it (there the arrays are complete once libenv_observe returns). get_state / set_state and
 * pgb200_set_consumer_output neither read nor write the rollout.
 * The cursor advances on the device, on the handle's stream, ahead of the step's render kernels: a step captured in
 * a CUDA graph after the first call fills successive slots at every replay; one captured before it never writes the
 * rollout. A handle without a rollout runs the kernels it ran before. A rollout of T steps plus the observation to
 * bootstrap from needs slots >= T + 1. */
struct pgb200_rollout {
    uint8_t *rgb;     /* [slots][num_envs][64][64][3] */
    float *rew;       /* [slots][num_envs] */
    uint8_t *first;   /* [slots][num_envs] */
    int32_t *cursor;  /* [1]: the slot the latest step (or the first call) wrote */
};
LIBENV_API int pgb200_get_rollout(libenv_env *handle, int slots, struct pgb200_rollout *out);

/* States of chosen envs in one call: get_state / set_state for the list envs[0, n) (host memory; the handle's own
 * indices), with the blobs in the same wire format, and no host round trip per env. On the device, each listed env's
 * header, generators, live entities, live grid cells and persistent scratch words are gathered into (or scattered
 * from) staging that a call grows up to 256 MiB, device and pinned each, and holds until libenv_close; the host
 * writes and reads the blobs from those records.
 * pgb200_get_states: the blob of envs[i] is (*data)[(*offsets)[i], (*offsets)[i + 1]). Both arrays are owned by
 * the handle and stay valid until the next pgb200_get_states on it, or libenv_close. Duplicate entries are allowed.
 * Waits for the step in flight, as get_state does, and performs the initial reset if it has not happened yet.
 * Returns 0, or -1 (nothing changed) for n < 0, an env out of range, or while the handle's stream is capturing.
 * pgb200_set_states: for each listed env, what set_state does: the blob data[offsets[i], offsets[i + 1]) is loaded,
 * the env's frame re-rendered and its rew, first and info slots rewritten from the restored state (with the consumer
 * output on, its current ring slot too). Envs not listed, the rollout, the pause mask, next_level_seed, final outputs,
 * the bank and lookahead slots are untouched. Every blob is read before any env changes; a malformed one is fatal,
 * `fatal: set_state: <check> (env <index>)`. Returns 0 once done, or -1 (nothing changed) for n < 0, an env out of
 * range, an env listed twice, or while the handle's stream is capturing. */
LIBENV_API int pgb200_get_states(libenv_env *handle, const int32_t *envs, int n, const char **data, const int64_t **offsets);
LIBENV_API int pgb200_set_states(libenv_env *handle, const int32_t *envs, int n, const char *data, const int64_t *offsets);

/* Snapshot slots: env states saved into and loaded from a store of `slots` slots on the device, without the host and
 * without the wire format, so that an RL loop can clone envs, branch a state into several envs, or return envs to
 * archived states inside its own device work (CUDA graphs included). Three int32 arrays of device memory (host memory
 * in the CPU debug build) control it, every entry -1 at first:
 *   save_from  [slots]     the caller's: at the next apply, slot s takes the state of env save_from[s]
 *   load_from  [num_envs]  the caller's: at the next apply, env e takes the state slot load_from[e] holds
 *   source     [slots]     read only: the env whose state slot s holds, -1 while it is empty
 * pgb200_apply_snapshots enqueues on the handle's stream, in this order:
 *   1. saves: every slot s with save_from[s] in [0, num_envs) takes that env's state; source[s] = that env and
 *      save_from[s] = -1;
 *   2. loads: every env e whose load_from[e] = s is a slot in [0, slots) that holds a state of e's own game
 *      (source[s] % G == e % G, G the games of the list) takes that state; load_from[e] = -1;
 *   3. every env loaded is observed as set_state observes it: its rgb, rew, first and info slots (and with the consumer
 *      output on, its current ring slot) are rewritten from the loaded state.
 * An entry that is not applied (an env or slot out of range, an empty slot, a slot of another game) keeps its value and
 * changes nothing. Saves run before loads, so one call can clone (save_from[s] = a, load_from[b] = s), and an env may
 * be saved and loaded in one call. After a load, env e's header (error bits, counters and high-water marks included),
 * both generators, live entities, live grid cells and persistent scratch words are a byte-for-byte copy of the source
 * env's at save time; so get_state(e) returns the blob get_state(source) returned then, and e steps on as the source
 * would have. Envs not loaded, the rollout, final outputs, the pause mask (a paused env loaded stays paused),
 * next_level_seed (pending overrides survive), the bank and lookahead slots (a slot keyed for the old state misses
 * once) are left alone; the peer mirror is refreshed by the next step. A slot holds the handle's own layout: it is not
 * portable across handles, builds or processes and is freed by libenv_close; get_state is the portable form.
 * pgb200_get_snapshots: *out = the arrays and the device bytes the store holds (slots of about 80 KB each for coinrun:
 * every slot is sized for the largest live state of the list). The first call performs the initial reset if it has not
 * happened yet, allocates the store, waits and returns 0; a later call with the same `slots` returns the same pointers.
 * Returns -1 (nothing changed) for slots < 1, a byte size that overflows, a failed allocation, a later call with other
 * `slots`, or a first call while the handle's stream is capturing.
 * pgb200_apply_snapshots: returns 0 once enqueued, or -1 on a handle without a store. It never waits for the host and
 * may be captured in a CUDA graph; each replay reads the arrays as they are then. Ordering as for next_level_seed:
 * write the arrays on the handle's stream before the call (with host buffers, the writes must be complete before the
 * call). pgb200_kernel_launches counts 2 + 2 * G per call: the save and load kernels, and each game's two frame
 * kernels (as set_state's observe, its camera kernel is not counted). */
struct pgb200_snapshots {
    int32_t *save_from;     /* [slots] */
    int32_t *load_from;     /* [num_envs] */
    const int32_t *source;  /* [slots] */
    int64_t bytes;          /* device memory the store holds */
};
LIBENV_API int pgb200_get_snapshots(libenv_env *handle, int slots, struct pgb200_snapshots *out);
LIBENV_API int pgb200_apply_snapshots(libenv_env *handle);

/* Re-home all subsequent work of this handle onto the caller's stream (a cudaStream_t, e.g. the
 * framework's current stream) so launches are ordered with the caller's own kernels and copies
 * without events. The handle's previous work is drained first. The value is used literally: NULL is
 * CUDA's legacy default stream. A new handle starts on a private non-blocking stream;
 * PGB200_PRIVATE_STREAM goes back to it. */
#define PGB200_PRIVATE_STREAM ((void *)(intptr_t)-1)
LIBENV_API void pgb200_set_stream(libenv_env *handle, void *stream);

/* Steps every env with the actions currently in the device action buffer. Asynchronous: enqueues
 * on the handle's stream and returns.
 *
 * CUDA graph capture. pgb200_act_device may be called while the handle's stream captures a CUDA graph
 * (cudaStreamBeginCapture, or pgb200_set_stream onto a stream that is capturing: that rebinding does not
 * wait). Every launch of the step, its ticket memsets and the fork to / join from the handle's auxiliary
 * streams become nodes of the caller's graph, and the consumer ring position advances on the device, so a
 * replay is the step issued at capture: same outputs as an eager call on the same inputs.
 * A captured step keeps what the host decided at capture: the launch shape (pgb200_set_launch_shape), the
 * level choice (the next_level_seed array is read only if pgb200_get_next_level_seeds had been called
 * before the capture; likewise the pause mask and pgb200_get_pause_mask, and the action repeat counts and
 * pgb200_get_action_repeat), the consumer output's buffer, dtype and k, and the handle's device buffers. Changing
 * any of these afterwards leaves the graph as it was; capture again. Replays of one handle's graphs must be
 * ordered with each other and with its eager work (one stream, or events). pgb200_kernel_launches counts
 * launches issued, a captured step once, not its replays. pgb200_apply_snapshots may be captured the same way.
 * Refused while the handle's stream is capturing (they wait for the device or allocate; -1, UINT32_MAX for
 * pgb200_get_errors, or a fatal message where the call returns nothing): the first
 * pgb200_get_next_level_seeds, pgb200_get_final_outputs, pgb200_get_pause_mask and pgb200_get_action_repeat,
 * pgb200_build_level_bank,
 * the first pgb200_enable_level_lookahead, pgb200_level_lookahead_info, the first pgb200_get_rollout, the first pgb200_get_snapshots, pgb200_get_device_buffers
 * before the initial reset, pgb200_set_consumer_output,
 * pgb200_set_rgb_mirror, get_state, set_state, pgb200_get_errors, pgb200_debug_cycles, pgb200_debug_read_env,
 * pgb200_set_launch_shape, pgb200_kernel_timing_begin / _end, pgb200_sync and the libenv_* calls. A step
 * cannot be captured with the peer mirror set (its parity is host state), with host buffers, or under
 * kernel timing: pgb200_act_device then ends the process with a message. */
LIBENV_API void pgb200_act_device(libenv_env *handle);

/* Blocks until all enqueued work of this handle is complete (VecGame::wait_for_stepping_threads). */
LIBENV_API void pgb200_sync(libenv_env *handle);

/* Per-env sticky error bits (0 = healthy): where the reference would fassert/exit, the device code
 * latches a bit instead. Copies num_envs words to `host_out`; returns the OR of all of them. */
LIBENV_API uint32_t pgb200_get_errors(libenv_env *handle, uint32_t *host_out);

/* Profiling aid: when the environment variable PGB200_DEBUG_TIMING is set at libenv_make time, the
 * logic kernel records each env's duration of the last step in SM cycles; copies num_envs words.
 * Returns -1 when timing was not enabled. */
LIBENV_API int pgb200_debug_cycles(libenv_env *handle, uint32_t *host_out);

/* Debug/inspection aid: copies env `env`'s header (512 B, layout csrc/pg_state.cuh EnvHdr) and up to
 * max_ents entity records (128 B each, csrc/pg_state.cuh Entity) to host memory; returns n_ents.
 * Returns -1 and copies nothing when env is outside [0, num_envs). */
LIBENV_API int pgb200_debug_read_env(libenv_env *handle, int env, void *hdr_out, void *ents_out, int max_ents);

/* Peer mirror for the single gather of a sharded run (SURVEY §8e, BASELINE configs[4]): mirror0 / mirror1
 * are device-accessible addresses (typically another GPU's memory mapped over NVLink: CUDA IPC or
 * torch symmetric memory) of this shard's [num_envs][64][64][3] slot in the gathered array. Every
 * step then copies each launch's frames there right behind its render kernel, alternating between
 * the two buffers step by step (pgb200_mirror_parity = the buffer the latest step wrote). Passing
 * NULL switches it off. The caller owns the synchronisation between ranks. Returns 0, or -1 in the
 * host debug build. */
LIBENV_API int pgb200_set_rgb_mirror(libenv_env *handle, void *mirror0, void *mirror1);
LIBENV_API int pgb200_mirror_parity(libenv_env *handle);

/* Consumer epilogue (SURVEY §8(f)4: the uint8 -> float normalise + frame-stack step that train-procgen style
 * learners run on every observation, README.md:13): a second output written by the render kernel.
 * `buffer` = device memory of [num_envs][slots][3][64][64] 16-bit floats, dtype 1 = fp16, 2 = bf16,
 * value = rgb / 255 (fp32 division, rounded to nearest even), planar CHW, slots = 1 for k_frames == 1
 * else 2*k_frames: the frame of step t goes to ring slots s = t mod k and s + k, so the ordered stack
 * (oldest first) is always the contiguous slot range [s + 1, s + k] (pgb200_consumer_slot = s). When
 * an env starts an episode the older frames of its window are zeroed (baselines' VecFrameStack). At
 * the call the current frames are written as step 0. buffer == NULL or dtype == 0 switches it off.
 * Returns 0, -1 on bad arguments or in the host debug build.
 * The ring position lives on the device (pgb200_get_consumer_slot_device) and every step advances it
 * there, ahead of its render kernels. pgb200_consumer_slot is the host's count of the steps issued since
 * the call, mod k: the device value as long as every step is issued by pgb200_act_device / libenv_act,
 * not by replaying a CUDA graph. */
LIBENV_API int pgb200_set_consumer_output(libenv_env *handle, void *buffer, int dtype, int k_frames);
LIBENV_API int pgb200_consumer_slot(libenv_env *handle);
/* `*out` = this handle's device-resident int32 ring position s of the consumer output (the slot the
 * latest step wrote), for a captured consumer that indexes the ring without the host: the ordered stack
 * is slots [s + 1, s + k]. Written on the handle's stream. Valid until libenv_close. Returns 0, or -1
 * in the host debug build. */
LIBENV_API int pgb200_get_consumer_slot_device(libenv_env *handle, int32_t **out);

/* Profiling variant only (-DPG_PHASE_TIMING): byte offset of the 12 phase-cycle counters inside the
 * header pgb200_debug_read_env returns; -1 in the product build. */
LIBENV_API int pgb200_debug_phase_offset(void);

/* Introspection: shared memory of one render CTA (the per-game frame) and the number of render CTAs
 * per SM the render kernel of `game` is compiled for. Returns -1 for an unknown game. */
LIBENV_API int pgb200_frame_info(const char *game, int *frame_bytes, int *ctas_per_sm);

/* Number of CUDA kernels this handle has launched so far (bench accounting): launches issued, so a step
 * captured in a CUDA graph counts once and its replays do not. */
LIBENV_API int64_t pgb200_kernel_launches(libenv_env *handle);

/* Per-kernel device timing for measurement (bench.py roofline): between begin and end every
 * (logic_kernel, setup_kernel, render_kernel) launch triple is bracketed by CUDA events on the stream it
 * runs on. end() synchronises and writes out[0] = sum of logic-kernel ms, out[1] = sum of render-kernel
 * ms, out[2] = number of launch triples timed, out[3] = env-steps those launches processed, out[4] =
 * sum of setup-kernel ms (out must hold 5 doubles); returns the number of triples. At most
 * max_launch_pairs triples are timed (further launches run untimed). Returns -1 on a handle with final
 * outputs (pgb200_get_final_outputs): the second phase of its steps is not bracketed by the triples. */
LIBENV_API int pgb200_kernel_timing_begin(libenv_env *handle, int max_launch_pairs);
/* Measurement knob: chunks > 0 forces that many env chunks per game and step (0 = the default
 * policy); serialize != 0 keeps every launch on the handle's stream, back to back, so a kernel's
 * event-timed duration is its own and not shared with kernels of other chunks. */
LIBENV_API void pgb200_set_launch_shape(libenv_env *handle, int chunks, int serialize);
LIBENV_API int pgb200_kernel_timing_end(libenv_env *handle, double *out);

/* 1 if this library was built for the GPU (the product), 0 for the CPU debug harness in tests/. */
LIBENV_API int pgb200_is_device_build(void);

#ifdef __cplusplus
}
#endif

#endif /* PROCGEN_B200_H */
