// get_state / set_state wire format (vecgame.cpp:437-457), byte-compatible with the reference:
// Game::serialize (game.cpp:170-229), BasicAbstractGame::serialize (basic-abstract-game.cpp:1169-1223),
// Entity::serialize (entity.cpp:90-131), RandGen::serialize (randgen.cpp:100-107: the libstdc++
// text form of std::mt19937), Grid::serialize (grid.h:69-73), buffer.h, and each game's tail
// (games/<name>.cpp serialize/deserialize, cited per game below).
//
// Host only. The env's records are copied out of HBM into a HostEnv, converted here, and copied
// back for set_state; nothing on the step path touches this file.
//
// Each record of the format is one function template over a wire: Save writes an env into a
// get_state blob, Load reads a set_state blob into an env. The order of the calls is the format;
// what only one direction does sits under `if constexpr (W::loading)` where it happens.
#pragma once
#include <iterator>
#include <stdexcept>
#include <string>
#include <type_traits>
#include <vector>

#include "pg_kernels.cuh"

namespace pg {
namespace host {

constexpr int SERIALIZE_VERSION = 0;  // game.h
constexpr int END_OF_BUFFER = 0xCAFECAFE;  // vecgame.cpp

struct HostEnv {
    EnvHdr h;
    std::vector<Entity> ents;     // ent_cap + 1 records (the last one is the agent's ghost slot)
    std::vector<int16_t> grid;    // grid_cap cells
    MT19937 rng, lvl_rng;
    std::vector<int32_t> scratch;
    int ent_cap = 0;
};

// options that are constant per VecGame and not kept per env on the device
struct ConstGameFields {
    int use_easy_jump = 0, plain_assets = 0, physics_mode = 0, game_type = 0;
};

// ---- buffer.h
struct WriteBuf {
    char *data;
    size_t offset = 0, length;
    WriteBuf(char *d, size_t n) : data(d), length(n) {}
    void need(size_t n) {
        if (offset + n > length)
            throw std::runtime_error("state buffer too small");
    }
    void write_int(int v) {
        need(4);
        memcpy(data + offset, &v, 4);
        offset += 4;
    }
    void write_bool(bool b) { write_int(b ? 1 : 0); }
    void write_float(float f) {
        need(4);
        memcpy(data + offset, &f, 4);
        offset += 4;
    }
    void write_string(const std::string &s) {
        write_int((int)s.size());
        need(s.size());
        memcpy(data + offset, s.data(), s.size());
        offset += s.size();
    }
};
struct ReadBuf {
    const char *data;
    size_t offset = 0, length;
    ReadBuf(const char *d, size_t n) : data(d), length(n) {}
    void need(size_t n) {
        if (offset + n > length)
            throw std::runtime_error("state buffer truncated");
    }
    int read_int() {
        need(4);
        int v;
        memcpy(&v, data + offset, 4);
        offset += 4;
        return v;
    }
    bool read_bool() { return read_int() > 0; }
    float read_float() {
        need(4);
        float f;
        memcpy(&f, data + offset, 4);
        offset += 4;
        return f;
    }
    std::string read_string() {
        int n = read_int();
        if (n < 0)
            throw std::runtime_error("bad string length in state");
        need((size_t)n);
        std::string s(data + offset, (size_t)n);
        offset += (size_t)n;
        return s;
    }
};

// ---- RandGen (randgen.cpp:100-114). libstdc++ prints the 624 state words and the position,
// separated by single spaces; its state is always a fully regenerated generation, ours twists
// words on demand (pg_rng.cuh), so the words [gen, 624) are brought up to date in a copy first.
inline std::string mt_to_text(const MT19937 &src) {
    MT19937 s = src;
    if (s.p < 624) {
        for (int k = s.gen; k < 624; k++) {
            const int k1 = (k + 1 == 624) ? 0 : k + 1;
            const int km = (k + 397 >= 624) ? k + 397 - 624 : k + 397;
            const uint32_t y = (s.mt[k] & 0x80000000u) | (s.mt[k1] & 0x7fffffffu);
            s.mt[k] = s.mt[km] ^ (y >> 1) ^ ((y & 1u) ? 0x9908b0dfu : 0u);
        }
    }
    std::string out;
    out.reserve(624 * 11 + 8);
    char tmp[16];
    for (int i = 0; i < 624; i++) {
        snprintf(tmp, sizeof(tmp), "%u ", s.mt[i]);
        out += tmp;
    }
    snprintf(tmp, sizeof(tmp), "%d", s.p);
    out += tmp;
    return out;
}
inline void mt_from_text(MT19937 &s, const std::string &text) {
    const char *p = text.c_str();
    char *end = nullptr;
    for (int i = 0; i < 624; i++) {
        unsigned long v = strtoul(p, &end, 10);
        if (end == p)
            throw std::runtime_error("bad mt19937 text in state");
        s.mt[i] = (uint32_t)v;
        p = end;
    }
    long pos = strtol(p, &end, 10);
    if (end == p || pos < 0 || pos > 624)
        throw std::runtime_error("bad mt19937 position in state");
    s.p = (int32_t)pos;
    s.gen = 624;  // every word of the imported generation is already regenerated
}

// ---- the two directions of the wire, one operation per kind of field:
//   i32, f32   a plain int32 (of any integer field) or float
//   boolean    a bool of a game's own (int32 on the device): written 0 / 1, read `> 0`
//   flag       a bool of Entity (uint8_t): written raw, read `!= 0`; so -1 reads back as 1 here, as 0 above
//   constant   written as given, read and dropped
//   expect     written as given, read and compared: a mismatch throws `err`
//   count      a length the env stores; read, it must lie in [0, cap]
//   length     the same for a length the env does not store: returns the number of entries to follow
//   mt         the text form of an MT19937
struct Save {  // get_state: env -> blob
    static constexpr bool loading = false;
    WriteBuf &b;
    template <class T>
    void i32(const T &v) { b.write_int((int)v); }
    void f32(float v) { b.write_float(v); }
    void boolean(int32_t v) { b.write_bool(v != 0); }
    void flag(uint8_t v) { b.write_int(v); }
    void constant(int v) { b.write_int(v); }
    void expect(int v, const char *) { b.write_int(v); }
    void expect(const std::string &s, const char *) { b.write_string(s); }
    int length(int n, int, const char *) {
        b.write_int(n);
        return n;
    }
    void count(int32_t n, int, const char *) { b.write_int(n); }
    void mt(const MT19937 &s) { b.write_string(mt_to_text(s)); }
};
struct Load {  // set_state: blob -> env, into the env as fetched, so what the blob does not carry keeps its value
    static constexpr bool loading = true;
    ReadBuf &b;
    template <class T>
    void i32(T &v) {
        static_assert(std::is_integral<T>::value, "i32 of a non-integer field");
        v = (T)b.read_int();
    }
    void f32(float &v) { v = b.read_float(); }
    void boolean(int32_t &v) { v = b.read_bool(); }
    void flag(uint8_t &v) { v = (uint8_t)(b.read_int() != 0); }
    void constant(int) { b.read_int(); }
    void expect(int v, const char *err) {
        if (b.read_int() != v)
            throw std::runtime_error(err);
    }
    void expect(const std::string &s, const char *err) {
        if (b.read_string() != s)
            throw std::runtime_error(err);
    }
    int length(int, int cap, const char *field) {
        const int n = b.read_int();
        if (n < 0 || n > cap)
            throw std::runtime_error("bad " + std::string(field) + " length " + std::to_string(n) + " (at most " +
                                     std::to_string(cap) + ")");
        return n;
    }
    void count(int32_t &n, int cap, const char *field) { n = length(n, cap, field); }
    void mt(MT19937 &s) { mt_from_text(s, b.read_string()); }
};

// p's bytes as a T, const when p is: the per-game tail and the scratch words hold typed records
template <class T, class U>
auto *view_as(U *p) {
    return reinterpret_cast<std::conditional_t<std::is_const<U>::value, const T, T> *>(p);
}
template <class T, class Env>
auto &tail(Env &e) {
    return *view_as<T>(e.h.game_state);
}

inline int find_entity_index(const HostEnv &e, int type) {  // basic-abstract-game.cpp:440-449
    int index = -1;
    for (int i = 0; i < e.h.n_ents; i++)
        if (e.ents[i].type == type)
            index = i;
    return index;
}

template <class W, class G>
void io_randgen(W &w, G &s) {  // randgen.cpp:100-114
    w.i32(s.seeded);
    w.mt(s);
}

template <class W, class E>
void io_entity(W &w, E &e) {  // entity.cpp:90-165
    if constexpr (W::loading)
        memset(&e, 0, sizeof(e));  // unlike the rest of the env, an entity keeps nothing of what it held
    w.f32(e.x);
    w.f32(e.y);
    w.f32(e.vx);
    w.f32(e.vy);
    w.f32(e.rx);
    w.f32(e.ry);
    w.i32(e.type);
    w.i32(e.image_type);
    w.i32(e.image_theme);
    w.i32(e.render_z);
    w.flag(e.will_erase);
    w.flag(e.collides_with_entities);
    w.f32(e.collision_margin);
    w.f32(e.rotation);
    w.f32(e.vrot);
    w.flag(e.is_reflected);
    w.i32(e.fire_time);
    w.i32(e.spawn_time);
    w.i32(e.life_time);
    w.i32(e.expire_time);
    w.flag(e.use_abs_coords);
    w.f32(e.friction);
    w.flag(e.smart_step);
    w.flag(e.avoids_collisions);
    w.flag(e.auto_erase);
    w.f32(e.alpha);
    w.f32(e.health);
    w.f32(e.theta);
    w.f32(e.grow_rate);
    w.f32(e.alpha_decay);
    w.f32(e.climber_spawn_x);
}

// ---- per-game tails. The device keeps a few derived values the reference recomputes or keeps
// outside the blob (entity indices instead of shared_ptrs, list lengths); set_state restores those too.
template <class W, class Env>
void io_tail(W &w, int game_id, Env &e) {
    switch (game_id) {
    case GAME_BIGFISH: {  // bigfish.cpp:169-173
        auto &s = tail<BigFishState>(e);
        w.i32(s.fish_eaten);
        w.f32(s.r_inc);
        break;
    }
    case GAME_BOSSFIGHT: {  // bossfight.cpp:415-476
        auto &s = tail<BossfightState>(e);
        w.count(s.n_attack_modes, (int)std::size(s.attack_modes), "attack_modes");
        for (int i = 0; i < s.n_attack_modes; i++) w.i32(s.attack_modes[i]);
        w.i32(s.last_fire_time);
        w.i32(s.time_to_swap);
        w.i32(s.invulnerable_duration);
        w.i32(s.vulnerable_duration);
        w.i32(s.num_rounds);
        w.i32(s.round_num);
        w.i32(s.round_health);
        w.i32(s.boss_vel_timeout);
        w.i32(s.curr_vel_timeout);
        w.i32(s.attack_mode);
        w.i32(s.player_laser_theme);
        w.i32(s.boss_laser_theme);
        w.i32(s.damaged_until_time);
        w.boolean(s.shields_are_up);
        w.boolean(s.barriers_moves_right);
        w.f32(s.base_fire_prob);
        w.f32(s.boss_bullet_vel);
        w.f32(s.barrier_vel);
        w.f32(s.barrier_spawn_prob);
        w.f32(s.rand_pct);
        w.f32(s.rand_fire_pct);
        w.f32(s.rand_pct_x);
        w.f32(s.rand_pct_y);
        if constexpr (W::loading) {
            s.boss_idx = find_entity_index(e, BossfightGame::BOSS);
            s.shields_idx = find_entity_index(e, BossfightGame::SHIELDS);
            if (s.boss_idx < 0 || s.shields_idx < 0)
                throw std::runtime_error("bossfight state without boss or shields");
        }
        break;
    }
    case GAME_CAVEFLYER:  // no fields of its own
        break;
    case GAME_CHASER: {  // chaser.cpp:388-398
        auto &s = tail<ChaserState>(e);
        auto *free_cells = e.scratch.data() + ChaserGame::MAZE_WORDS;
        auto *is_space = free_cells + ChaserGame::LIST_WORDS;
        w.count(s.n_free_cells, ChaserGame::LIST_WORDS, "free_cells");
        for (int i = 0; i < s.n_free_cells; i++) w.i32(free_cells[i]);
        const int n = w.length(e.h.grid_size, ChaserGame::LIST_WORDS, "is_space_vec");
        for (int i = 0; i < n; i++) w.boolean(is_space[i]);
        w.i32(s.eat_timeout);
        w.i32(s.egg_timeout);
        w.i32(s.eat_time);
        w.i32(s.total_enemies);
        w.i32(s.total_orbs);
        w.i32(s.orbs_collected);
        w.i32(s.maze_dim);
        break;
    }
    case GAME_CLIMBER: {  // climber.cpp serialize
        auto &s = tail<ClimberState>(e);
        w.boolean(s.has_support);
        w.boolean(s.facing_right);
        w.i32(s.coin_quota);
        w.i32(s.coins_collected);
        w.i32(s.wall_theme);
        w.f32(s.gravity);
        w.f32(s.air_control);
        break;
    }
    case GAME_COINRUN: {  // coinrun.cpp:500-509
        auto &s = tail<CoinRunState>(e);
        w.f32(s.last_agent_y);
        w.i32(s.wall_theme);
        w.boolean(s.has_support);
        w.boolean(s.facing_right);
        w.boolean(s.is_on_crate);
        w.f32(s.gravity);
        w.f32(s.air_control);
        break;
    }
    case GAME_DODGEBALL: {  // dodgeball.cpp:442-451
        auto &s = tail<DodgeballState>(e);
        w.f32(s.min_dim);
        w.f32(s.hard_min_dim);
        w.f32(s.ball_vscale);
        w.f32(s.ball_r);
        w.i32(s.last_fire_time);
        w.i32(s.num_enemies);
        w.i32(s.enemy_fire_delay);
        break;
    }
    case GAME_FRUITBOT: {  // fruitbot.cpp serialize
        auto &s = tail<FruitBotState>(e);
        w.f32(s.min_dim);
        w.f32(s.bullet_vscale);
        w.i32(s.last_fire_time);
        break;
    }
    case GAME_HEIST: {  // heist.cpp:211-216: num_keys, then has_keys as a vector with its own length
        auto &s = tail<HeistState>(e);
        w.i32(s.num_keys);
        w.i32(s.world_dim);
        const int n = w.length(s.num_keys, (int)std::size(s.has_keys), "has_keys");
        for (int i = 0; i < n; i++) w.boolean(s.has_keys[i]);
        break;
    }
    case GAME_JUMPER: {  // jumper.cpp:445-469
        auto &s = tail<JumperState>(e);
        w.i32(s.jump_count);
        w.i32(s.jump_delta);
        w.i32(s.jump_time);
        w.boolean(s.has_support);
        w.boolean(s.facing_right);
        w.i32(s.wall_theme);
        w.f32(s.compass_dim);
        if constexpr (W::loading) {
            s.goal_idx = find_entity_index(e, JumperGame::GOAL);
            if (s.goal_idx < 0)
                throw std::runtime_error("jumper state without a goal");
        }
        break;
    }
    case GAME_LEAPER: {  // leaper.cpp serialize
        auto &s = tail<LeaperState>(e);
        w.i32(s.bottom_road_y);
        w.count(s.n_road, (int)std::size(s.road_lane_speeds), "road_lane_speeds");
        for (int i = 0; i < s.n_road; i++) w.f32(s.road_lane_speeds[i]);
        w.i32(s.bottom_water_y);
        w.count(s.n_water, (int)std::size(s.water_lane_speeds), "water_lane_speeds");
        for (int i = 0; i < s.n_water; i++) w.f32(s.water_lane_speeds[i]);
        w.i32(s.goal_y);
        break;
    }
    case GAME_MAZE: {  // maze.cpp serialize
        auto &s = tail<MazeState>(e);
        w.i32(s.maze_dim);
        w.i32(s.world_dim);
        break;
    }
    case GAME_MINER:  // miner.cpp serialize
        w.i32(tail<MinerState>(e).diamonds_remaining);
        break;
    case GAME_NINJA: {  // ninja.cpp serialize
        auto &s = tail<NinjaState>(e);
        w.boolean(s.has_support);
        w.boolean(s.facing_right);
        w.i32(s.last_fire_time);
        w.i32(s.wall_theme);
        w.f32(s.gravity);
        w.f32(s.air_control);
        w.f32(s.jump_charge);
        w.f32(s.jump_charge_inc);
        break;
    }
    case GAME_PLUNDER: {  // plunder.cpp:243-259: four vectors with their own lengths, then num_lanes
        auto &s = tail<PlunderState>(e);
        w.i32(s.last_fire_time);
        int n = w.length(s.num_lanes, (int)std::size(s.lane_directions), "lane_directions");
        for (int i = 0; i < n; i++) w.boolean(s.lane_directions[i]);
        n = w.length(6, (int)std::size(s.target_bools), "target_bools");
        for (int i = 0; i < n; i++) w.boolean(s.target_bools[i]);
        n = w.length(6, (int)std::size(s.image_permutation), "image_permutation");
        for (int i = 0; i < n; i++) w.i32(s.image_permutation[i]);
        n = w.length(s.num_lanes, (int)std::size(s.lane_vels), "lane_vels");
        for (int i = 0; i < n; i++) w.f32(s.lane_vels[i]);
        w.i32(s.num_lanes);
        w.i32(s.num_current_ship_types);
        w.i32(s.targets_hit);
        w.i32(s.target_quota);
        w.f32(s.juice_left);
        w.f32(s.r_scale);
        w.f32(s.spawn_prob);
        w.f32(s.legend_r);
        w.f32(s.min_agent_x);
        break;
    }
    case GAME_STARPILOT: {  // starpilot.cpp:451-461: the remaining spawners, in list order. set_state lays them
                            // out in that order; init_hps is replayed by the caller on the device side: it
                            // depends only on the distribution mode, whose values are already in the tail
        auto &s = tail<StarpilotState>(e);
        auto *recs = view_as<Entity>(e.scratch.data());
        auto *order = e.scratch.data() + StarpilotGame::MAX_SPAWNERS * StarpilotGame::ENT_WORDS;
        w.count(s.n_spawners, StarpilotGame::MAX_SPAWNERS, "spawners");
        for (int i = 0; i < s.n_spawners; i++) {
            if constexpr (W::loading)
                order[i] = i;
            io_entity(w, recs[order[i]]);
        }
        break;
    }
    default:
        throw std::runtime_error("unknown game id");
    }
}

// ---- Game + BasicAbstractGame
template <class W, class Env>
void io_env(W &w, const char *game_name, int game_id, Env &e, const ConstGameFields &cf) {
    auto &h = e.h;
    w.expect(SERIALIZE_VERSION, "serialize version mismatch");
    w.expect(game_name, "state belongs to another game");
    w.i32(h.options.paint_vel_info);
    w.i32(h.options.use_generated_assets);
    w.i32(h.options.use_monochrome_assets);
    w.i32(h.options.restrict_themes);
    w.i32(h.options.use_backgrounds);
    w.i32(h.options.center_agent);
    w.i32(h.options.debug_mode);
    w.i32(h.options.distribution_mode);
    w.i32(h.options.use_sequential_levels);
    if constexpr (W::loading)
        if (h.options.use_generated_assets)
            throw std::runtime_error("use_generated_assets is not supported");
    w.constant(cf.use_easy_jump);  // the per-VecGame constants: set_state keeps the handle's
    w.constant(cf.plain_assets);
    w.constant(cf.physics_mode);
    w.i32(h.grid_step);
    w.i32(h.level_seed_low);
    w.i32(h.level_seed_high);
    w.constant(cf.game_type);
    w.i32(h.game_n);
    io_randgen(w, e.lvl_rng);
    io_randgen(w, e.rng);
    w.f32(h.reward);
    w.i32(h.done);
    w.i32(h.level_complete);
    w.i32(h.action);
    w.i32(h.timeout);
    w.i32(h.current_level_seed);
    w.i32(h.prev_level_seed);
    w.i32(h.episodes_remaining);
    w.i32(h.episode_done);
    w.i32(h.last_reward_timer);
    w.f32(h.last_reward);
    w.i32(h.default_action);
    w.i32(h.fixed_asset_seed);
    w.i32(h.cur_time);
    w.constant(0);  // is_waiting_for_step: get_state waits for the step first
    // BasicAbstractGame
    w.i32(h.grid_size);
    if constexpr (!W::loading)
        if (h.agent_idx >= e.ent_cap)
            throw std::runtime_error("the agent is not in the entity list");
    w.count(h.n_ents, e.ent_cap, "entities");
    for (int i = 0; i < h.n_ents; i++) io_entity(w, e.ents[i]);
    if constexpr (W::loading) {
        if (h.max_ents_seen < h.n_ents)
            h.max_ents_seen = h.n_ents;
        h.agent_idx = find_entity_index(e, PLAYER);  // basic-abstract-game.cpp:1231-1233
        if (h.agent_idx < 0)
            throw std::runtime_error("state without an agent");
    }
    w.constant(0);  // use_procgen_background: every game loads real backgrounds (basic-abstract-game.cpp:54-66)
    w.i32(h.background_index);
    w.f32(h.bg_tile_ratio);
    w.f32(h.bg_pct_x);
    w.f32(h.char_dim);
    w.i32(h.last_move_action);
    w.i32(h.move_action);
    w.i32(h.special_action);
    w.f32(h.mixrate);
    w.f32(h.maxspeed);
    w.f32(h.max_jump);
    w.f32(h.action_vx);
    w.f32(h.action_vy);
    w.f32(h.action_vrot);
    w.f32(h.center_x);
    w.f32(h.center_y);
    w.i32(h.random_agent_start);
    w.i32(h.has_useful_vel_info);
    w.i32(h.step_rand_int);
    {
        // asset_rand_gen: only the generated-asset path ever seeds or draws from it, so get_state writes
        // the default-constructed engine (std::mt19937 default seed 5489) and set_state reads one and drops it
        MT19937 asset;
        memset(&asset, 0, sizeof(asset));
        mt_seed(asset, 5489u);
        asset.seeded = 0;
        io_randgen(w, asset);
    }
    w.i32(h.main_width);
    w.i32(h.main_height);
    w.i32(h.out_of_bounds_object);
    w.f32(h.unit);
    w.f32(h.view_dim);
    w.f32(h.x_off);
    w.f32(h.y_off);
    w.f32(h.visibility);
    w.f32(h.min_visibility);
    // Grid<int>::serialize (grid.h:69-73): the world's size once more, then its cells
    int gw = h.main_width, gh = h.main_height, cells = gw * gh;
    w.i32(gw);
    w.i32(gh);
    w.i32(cells);
    if constexpr (W::loading)
        if (gw != h.main_width || gh != h.main_height || cells != gw * gh || cells > (int)e.grid.size())
            throw std::runtime_error("grid does not fit this build's capacity for the game");
    for (int i = 0; i < cells; i++) w.i32(e.grid[i]);
    io_tail(w, game_id, e);
    w.expect(END_OF_BUFFER, "trailing bytes in state");
}

inline void serialize_env(const char *game_name, int game_id, const HostEnv &e, const ConstGameFields &cf, WriteBuf &b) {
    Save w{b};
    io_env(w, game_name, game_id, e, cf);
}

// the per-VecGame constants of the blob are read and dropped, so any ConstGameFields will do
inline void deserialize_env(const char *game_name, int game_id, HostEnv &e, ReadBuf &b) {
    Load w{b};
    io_env(w, game_name, game_id, e, ConstGameFields{});
}

}  // namespace host
}  // namespace pg
