// StarPilot on the device engine. Behaviour restated from games/starpilot.cpp (cited per function).
#pragma once
#include "../pg_raster.cuh"
#include "../pg_stdsort.cuh"

namespace pg {

struct StarpilotState {
    float hp_vs[9], hp_healths[9], hp_bullet_r[9], hp_object_r[9], hp_object_prob_weight[9];
    float total_prob_weight, hp_slow_v, hp_weapon_bullet_dist, hp_spawn_right_threshold;
    int32_t hp_min_enemy_delta_t, hp_max_group_size, hp_max_enemy_delta_t;
    int32_t n_spawners;  // live length of the sorted spawner list (popped from the back)
};

struct StarpilotGame : Defaults<StarpilotGame>, DrawDefaults<StarpilotGame> {
    using E = Engine<StarpilotGame>;
    static constexpr int ENT_CAP = 256;
    static constexpr int GRID_CAP = 16 * 16;
    // the spawner list (starpilot.cpp:33): <= 49 groups x 5 ships; full Entity records in creation
    // order, then the sorted order as indices into them
    static constexpr int MAX_SPAWNERS = 256;
    static constexpr int ENT_WORDS = (int)(sizeof(Entity) / 4);
    static constexpr int SCRATCH_WORDS = MAX_SPAWNERS * ENT_WORDS + MAX_SPAWNERS;
    static constexpr int PERSIST_SCRATCH_FIRST = 0;  // the spawner list
    static constexpr int PERSIST_SCRATCH_WORDS = SCRATCH_WORDS;
    static constexpr int MAX_VISIBLE_ENTS = 256;
    static constexpr int MAX_ROT_BLITS = 224;  // ships, bullets and the agent all carry a rotation
    static constexpr int MAX_VIEW_CELLS = 16;
    static constexpr const char *NAME = "starpilot";
    static constexpr bool DEFER_ROTATED = true;
    static constexpr bool DRAWS_GRID = false;  // entities only; the grid stays all SPACE
    // is_blocked / is_blocked_ents / will_reflect are the engine defaults here: only an entity typed WALL_OBJ or as the out-of-bounds object could block
    static PG_HD bool may_be_obstacle(Ctx &c, int t) { return t == WALL_OBJ || t == c.oob; }
    static PG_HD bool may_block_or_reflect(Ctx &c, int src, int t) { return may_be_obstacle(c, t); }

    // starpilot.cpp:6-26
    static constexpr float V_SCALE = 2.0f / 5.0f;
    static constexpr float BG_RATIO = 18;
    static constexpr float ENEMY_REWARD = 1.0f, COMPLETION_BONUS = 10.0f;
    static constexpr int BULLET_PLAYER = 1, BULLET2 = 2, BULLET3 = 3, FLYER = 4, METEOR = 5, CLOUD = 6, TURRET = 7, FAST_FLYER = 8, FINISH_LINE = 9;
    static constexpr int SHOOTER_WIN_TIME = 500, NUM_BASIC_OBJECTS = 9, NUM_SHIP_THEMES = 7;

    static PG_HD StarpilotState &st(Ctx &c) { return game_state<StarpilotState>(c); }
    static PG_HD Entity *spawner_recs(Ctx &c) { return reinterpret_cast<Entity *>(c.scratch); }
    static PG_HD int32_t *spawner_order(Ctx &c) { return c.scratch + MAX_SPAWNERS * ENT_WORDS; }

    // starpilot.cpp:49-53
    static PG_HD void init_constants(Ctx &c) {
        base_init_constants(c);
        c.h->main_width = 16;
        c.h->main_height = 16;
    }
    // starpilot.cpp:110-129: black, then the background tiled 18 times sideways and scrolled with time
    template <class Frame>
    static PG_HD void make_background_blits(Ctx &c, Frame &f) {
        EnvHdr &h = *c.h;
        f.n_bg = 0;
        if (!h.options.use_backgrounds)
            return;
        float scale = (float)(RES_H / h.main_height);
        float bg_k = 3;
        float t = (float)h.cur_time;
        float x_off = -t * scale * st(c).hp_slow_v * 2 / h.char_dim;
        double r_bg[4] = {(double)x_off, (double)(-RES_H * (bg_k - 1) / 2), (double)(RES_H * bg_k * BG_RATIO), (double)(RES_H * bg_k)};
        SpriteDesc bg = c.assets->backgrounds[h.background_index];
        const int nt = Raster<StarpilotGame, Frame>::tile_count(r_bg, 1);
        int n = 0;
        for (int i = 0; i < nt; i++) {
            double tr[4];
            Raster<StarpilotGame, Frame>::tile_rect(r_bg, 1, nt, i, tr);
            Blit b;
            make_image_blit(b, tr[0], tr[1], tr[2], tr[3], bg, false, 256, f.snap != 0);
            if (b.kind == BLIT_NONE)
                continue;  // tile entirely off screen
            if (n < MAX_BG_BLITS)
                f.bg[n++] = b;
            else
                h.err |= ERR_BLIT_OVERFLOW;
        }
        f.n_bg = n;
    }
    // starpilot.cpp:364-372
    static PG_HD bool is_lethal(int type) {
        return type == FLYER || type == FAST_FLYER || type == BULLET2 || type == BULLET3 || type == TURRET || type == METEOR;
    }
    static PG_HD bool is_destructible(int type) { return type == FLYER || type == FAST_FLYER || type == TURRET || type == METEOR; }
    // starpilot.cpp:131-141
    static PG_HD void handle_agent_collision(Ctx &c, int oi) {
        int t = c.ents[oi].type;
        if (t == FINISH_LINE) {
            c.h->done = 1;
            c.h->reward += COMPLETION_BONUS;
            c.h->level_complete = 1;
        } else if (is_lethal(t)) {
            c.h->done = 1;
        }
    }
    // starpilot.cpp:143-150
    static PG_HD void handle_collision(Ctx &c, int si, int ti) {
        Entity &src = c.ents[si];
        Entity &target = c.ents[ti];
        if (src.type == BULLET_PLAYER && target.type != CLOUD && is_destructible(target.type)) {
            src.will_erase = 1;
            target.health -= 1;
            float sx = src.x, sy = src.y, tvx = target.vx, tvy = target.vy, r = (float)(.5 * src.rx);
            E::add_entity(c, sx, sy, tvx, tvy, r, EXPLOSION);
        }
    }
    // starpilot.cpp:152-232
    static PG_HD void init_hps(Ctx &c) {
        StarpilotState &s = st(c);
        EnvHdr &h = *c.h;
        float scale = 1;
        for (int i = 0; i < NUM_BASIC_OBJECTS; i++) {
            s.hp_vs[i] = 1;
            s.hp_healths[i] = 0;
            s.hp_object_prob_weight[i] = 1;
            s.hp_object_r[i] = scale / 2;
        }
        float default_bullet_r = (float)(scale / 2.5);
        const int mode = h.options.distribution_mode;
        if (mode == EasyMode) {
            s.hp_object_prob_weight[METEOR] = 0;
            s.hp_object_prob_weight[CLOUD] = 0;
            s.hp_object_prob_weight[TURRET] = 0;
            s.hp_object_prob_weight[FAST_FLYER] = 0;
            s.hp_vs[FLYER] = .75;
            s.hp_vs[BULLET2] = 1.25;
            s.hp_healths[TURRET] = 5;
            s.hp_healths[FLYER] = 2;
            s.hp_healths[FAST_FLYER] = 1;
            h.maxspeed = 0.75;
        } else if (mode == HardMode) {
            s.hp_vs[BULLET2] = 2;
            s.hp_healths[TURRET] = 5;
            s.hp_healths[FLYER] = 2;
            s.hp_healths[FAST_FLYER] = 1;
            h.maxspeed = 0.75;
        } else if (mode == ExtremeMode) {
            s.hp_vs[BULLET2] = 2;
            s.hp_healths[TURRET] = 10;
            s.hp_healths[FLYER] = 5;
            s.hp_healths[FAST_FLYER] = 2;
            h.maxspeed = 0.5;
            default_bullet_r = scale / 5;
        } else {
            h.err |= ERR_FASSERT;
        }
        for (int i = 0; i < NUM_BASIC_OBJECTS; i++) s.hp_bullet_r[i] = default_bullet_r;
        s.hp_healths[METEOR] = 500;
        s.hp_vs[FAST_FLYER] = 1.5;
        s.hp_vs[BULLET_PLAYER] = 2;
        s.hp_vs[BULLET3] = 2;
        s.hp_object_r[TURRET] = scale * 2;
        s.hp_object_r[METEOR] = scale * 2;
        s.hp_object_r[CLOUD] = scale * 2;
        s.hp_object_prob_weight[FLYER] = 3;
        s.hp_slow_v = .5;
        s.hp_max_group_size = 5;
        s.hp_weapon_bullet_dist = 3;
        s.hp_min_enemy_delta_t = 10;
        s.hp_max_enemy_delta_t = s.hp_min_enemy_delta_t + 20;
        s.hp_spawn_right_threshold = 0.9f;
        s.hp_object_prob_weight[BULLET_PLAYER] = 0;
        s.hp_object_prob_weight[BULLET2] = 0;
        s.hp_object_prob_weight[BULLET3] = 0;
        s.total_prob_weight = 0;
        for (int i = 2; i < NUM_BASIC_OBJECTS; i++) s.total_prob_weight += s.hp_object_prob_weight[i];
    }
    // starpilot.cpp:234-342 — cos/sin are the double overloads
    static PG_HD void add_spawners(Ctx &c) {
        StarpilotState &s = st(c);
        EnvHdr &h = *c.h;
        MT19937 &rg = *c.rng;
        Entity *recs = spawner_recs(c);
        int t = 1 + rand_randint(rg, s.hp_min_enemy_delta_t, s.hp_max_enemy_delta_t);
        bool can_spawn_left = h.options.distribution_mode != EasyMode;
        for (int i = 0; t <= SHOOTER_WIN_TIME; i++) {
            int group_size = 1;
            float start_weight = rand_rand01(rg) * s.total_prob_weight;
            float curr_weight = start_weight;
            int type;
            for (type = 2; type < NUM_BASIC_OBJECTS; type++) {
                curr_weight -= s.hp_object_prob_weight[type];
                if (curr_weight <= 0)
                    break;
            }
            if (type >= NUM_BASIC_OBJECTS)
                type = NUM_BASIC_OBJECTS - 1;
            float r = s.hp_object_r[type];
            int flyer_theme = 0;
            if (type == FLYER || type == FAST_FLYER) {
                group_size = rand_randint(rg, 0, s.hp_max_group_size) + 1;
                flyer_theme = rand_randn(rg, NUM_SHIP_THEMES);
            }
            float y_pos = E::rand_pos(c, r, 0, (float)h.main_height);
            for (int j = 0; j < group_size; j++) {
                int spawn_time = t + j * 5;
                int fire_time = rand_randint(rg, 10, 100);
                float k = 2 * PI_F / 4;
                float theta = (float)(((double)rand_rand01(rg) - .5) * (double)k);
                float v_scale = s.hp_vs[type];
                if (rand_randint(rg, 0, 2) == 1)
                    theta = 0;
                float health = s.hp_healths[type];
                if (type == METEOR || type == CLOUD) {
                    theta = 0;
                    v_scale = s.hp_slow_v;
                    fire_time = -1;
                } else if (type == TURRET) {
                    theta = 0;
                    v_scale = s.hp_slow_v;
                    fire_time = rand_randint(rg, 20, 30);
                }
                v_scale *= V_SCALE;
                float vx = (float)(-1 * cos((double)theta) * (double)v_scale);
                float vy = (float)(sin((double)theta) * (double)v_scale);
                bool spawn_right = true;
                float x_pos;
                if (type == FLYER || type == FAST_FLYER) {
                    if (rand_rand01(rg) > s.hp_spawn_right_threshold && can_spawn_left)
                        spawn_right = false;
                }
                if (spawn_right) {
                    x_pos = h.main_width + r;
                } else {
                    x_pos = -r;
                    vx *= -1;
                }
                if (s.n_spawners >= MAX_SPAWNERS) {
                    h.err |= ERR_SCRATCH_OVERFLOW;
                    continue;
                }
                Entity &sp = recs[s.n_spawners++];
                entity_init(sp, x_pos, y_pos, vx, vy, r, r, type);
                sp.fire_time = fire_time;
                sp.spawn_time = spawn_time;
                sp.health = health;
                if (type == CLOUD) {
                    sp.render_z = 1;
                    E::choose_random_theme(c, sp);
                } else if (type == METEOR) {
                    E::choose_random_theme(c, sp);
                } else if (type == FLYER || type == FAST_FLYER) {
                    sp.image_theme = flyer_theme;
                    sp.rotation = ((vx > 0) ? -1 : 1) * PI_F / 2;
                } else if (type == TURRET) {
                    E::choose_random_theme(c, sp);
                    E::match_aspect_ratio(c, sp);
                }
            }
            t += rand_randint(rg, s.hp_min_enemy_delta_t, s.hp_max_enemy_delta_t);
        }
    }
    // starpilot.cpp:344-362
    static PG_HD void game_reset(Ctx &c) {
        E::basic_game_reset(c);
        c.h->options.center_agent = 0;
        init_hps(c);
        StarpilotState &s = st(c);
        s.n_spawners = 0;
        add_spawners(c);
        // std::sort(spawners, spawn_cmp) with spawn_cmp(x, y) = x->spawn_time > y->spawn_time
        // (starpilot.cpp:28-30, 356): not stable, so the library's exact algorithm is replayed
        int32_t *order = spawner_order(c);
        for (int i = 0; i < s.n_spawners; i++) order[i] = i;
        const Entity *recs = spawner_recs(c);
        pg_std_sort(order, s.n_spawners, [recs](int32_t x, int32_t y) { return recs[x].spawn_time > recs[y].spawn_time; });
        agent_of(c).rotation = PI_F / 2;
        E::choose_random_theme(c, agent_of(c));
    }
    // starpilot.cpp:374-384
    static PG_HD bool should_fire(const Entity &e1, int cur_time) {
        if (e1.fire_time <= 0)
            return false;
        if (e1.type == TURRET)
            return (cur_time - e1.spawn_time) % e1.fire_time == 0;
        return cur_time - e1.spawn_time == e1.fire_time;
    }
    // starpilot.cpp:386-449
    static PG_HD void game_step(Ctx &c) {
        E::basic_game_step(c);
        EnvHdr &h = *c.h;
        StarpilotState &s = st(c);
        bool is_firing = h.special_action != 0;
        for (int i = h.n_ents - 1; i >= 0; i--) {
            if (c.ents[i].type == PLAYER)
                continue;
            if (should_fire(c.ents[i], h.cur_time)) {
                const Entity m = c.ents[i];
                const Entity &a = agent_of(c);
                int bullet_type = m.type == TURRET ? BULLET3 : BULLET2;
                float bullet_r = s.hp_bullet_r[m.type];
                float b_vx = a.x - m.x;
                float b_vy = a.y - m.y;
                float bv_scale = (float)((double)(s.hp_vs[bullet_type] * V_SCALE) / pg_dsqrt((double)(b_vx * b_vx + b_vy * b_vy)));
                b_vx = b_vx * bv_scale;
                b_vy = b_vy * bv_scale;
                int bi = E::add_entity(c, m.x, m.y, b_vx, b_vy, bullet_r, bullet_type);
                entity_face_direction(c.ents[bi], b_vx, b_vy, -1 * PI_F / 2);
            }
            Entity &m = c.ents[i];
            if (m.health <= 0 && is_destructible(m.type) && !m.will_erase) {
                E::spawn_child(c, i, EXPLOSION, (float)(.5 * m.rx), true);
                h.reward += ENEMY_REWARD;
                c.ents[i].will_erase = 1;
            }
        }
        {
            const Entity *recs = spawner_recs(c);
            const int32_t *order = spawner_order(c);
            while (s.n_spawners > 0 && h.cur_time == recs[order[s.n_spawners - 1]].spawn_time) {
                int ei = E::push_entity(c);
                c.ents[ei] = recs[order[s.n_spawners - 1]];
                s.n_spawners--;
            }
        }
        float bullet_r = s.hp_bullet_r[PLAYER];
        if (is_firing) {
            float theta = h.special_action == 2 ? PI_F : 0;
            float v_scale = s.hp_vs[BULLET_PLAYER] * V_SCALE;
            float vx = (float)(cos((double)theta) * (double)v_scale);
            float vy = (float)(sin((double)theta) * (double)v_scale);
            const Entity &a = agent_of(c);
            float x_off = (float)((double)a.rx * cos((double)theta));
            int bi = E::add_entity(c, a.x + x_off, a.y, vx, vy, bullet_r, BULLET_PLAYER);
            c.ents[bi].collides_with_entities = 1;
            entity_face_direction(c.ents[bi], vx, vy);
            c.ents[bi].rotation -= PI_F / 2;
        }
        if (h.cur_time == SHOOTER_WIN_TIME) {
            int fi = E::add_entity_rxy(c, (float)h.main_width, (float)(h.main_height / 2), -1 * s.hp_slow_v * V_SCALE, 0, 2, (float)(h.main_height / 2), FINISH_LINE);
            Entity &finish = c.ents[fi];
            E::choose_random_theme(c, finish);
            E::match_aspect_ratio(c, finish, false);
            finish.x = h.main_width + finish.rx;
        }
    }
};

}  // namespace pg
