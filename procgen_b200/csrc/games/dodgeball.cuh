// Dodgeball on the device engine. Behaviour restated from games/dodgeball.cpp (cited per function).
#pragma once
#include "../pg_raster.cuh"

namespace pg {

struct DodgeballState {
    float min_dim, hard_min_dim, ball_vscale, ball_r;
    int32_t last_fire_time, num_enemies, enemy_fire_delay;
    int32_t n_rooms;  // the room list itself (x, y, w, h floats) lives in the env's scratch words
};

struct DodgeballGame : Defaults<DodgeballGame>, DrawDefaults<DodgeballGame> {
    using E = Engine<DodgeballGame>;
    static constexpr int ENT_CAP = 160;
    static constexpr int GRID_CAP = 40 * 40;
    static constexpr int MAX_ROOMS = 64;  // <= 1 + 2 * 16 splits
    static constexpr int SCRATCH_WORDS = 4 * MAX_ROOMS;
    static constexpr int PERSIST_SCRATCH_FIRST = 0;  // the room list
    static constexpr int PERSIST_SCRATCH_WORDS = SCRATCH_WORDS;
    static constexpr int MAX_VISIBLE_ENTS = 256;  // lava walls are tiled; only the on-screen run of tiles becomes blits (measured peak 119)
    static constexpr int MAX_ROT_BLITS = 64;      // everything that faces a direction or spins (measured peak 20)
    static constexpr int MAX_VIEW_CELLS = 20;
    static constexpr const char *NAME = "dodgeball";
    static constexpr bool DEFER_ROTATED = true;

    // dodgeball.cpp:8-24
    static constexpr float COMPLETION_BONUS = 10.0f;
    static constexpr int LAVA_WALL = 1, PLAYER_BALL = 3, ENEMY = 4, DOOR = 5, ENEMY_BALL = 6, DOOR_OPEN = 7, DUST_CLOUD = 8, OOB_WALL = 10;
    static constexpr int ENEMY_REWARD = 2;
    static constexpr int NUM_ENEMY_THEMES = 7;
    static constexpr float ENEMY_VEL = 0.05f;
    static constexpr float BALL_V_ROT = PI_F * 0.23f;

    static PG_HD DodgeballState &st(Ctx &c) { return game_state<DodgeballState>(c); }
    static PG_HD float *room(Ctx &c, int i) { return reinterpret_cast<float *>(c.scratch) + 4 * i; }

    // dodgeball.cpp:37-44
    static PG_HD void init_constants(Ctx &c) {
        base_init_constants(c);
        c.h->mixrate = .5;
        c.h->out_of_bounds_object = OOB_WALL;
        st(c).enemy_fire_delay = 50;
    }
    // dodgeball.cpp:90-96
    static PG_HD int image_for_type(Ctx &c, int type) {
        if (type == DOOR)
            return st(c).num_enemies == 0 ? DOOR_OPEN : DOOR;
        return type < 0 ? -type : type;
    }
    // dodgeball.cpp:98-100
    static PG_HD bool will_reflect(Ctx &c, int src, int target) {
        return src == ENEMY && (target == LAVA_WALL || target == c.oob);
    }
    // no entity ever carries WALL_OBJ or the out-of-bounds id, so entity overlaps only matter for
    // an enemy bouncing off lava
    static PG_HD bool may_be_obstacle(Ctx &c, int target) { return target == LAVA_WALL; }
    static PG_HD bool may_block_or_reflect(Ctx &c, int src, int target) { return src == ENEMY && target == LAVA_WALL; }
    // dodgeball.cpp:102-118
    static PG_HD void handle_agent_collision(Ctx &c, int oi) {
        int t = c.ents[oi].type;
        if (t == ENEMY || t == ENEMY_BALL || t == LAVA_WALL) {
            c.h->done = 1;
        } else if (t == DOOR) {
            if (st(c).num_enemies == 0) {
                c.h->done = 1;
                c.h->reward += COMPLETION_BONUS;
                c.h->level_complete = 1;
            }
        }
    }
    // dodgeball.cpp:120-151
    static PG_HD void handle_collision(Ctx &c, int si, int ti) {
        Entity &src = c.ents[si];
        Entity &target = c.ents[ti];
        if (target.type == PLAYER_BALL) {
            if (src.type == LAVA_WALL) {
                target.will_erase = 1;
            } else if (src.type == ENEMY) {
                src.health -= 1;
                target.will_erase = 1;
                if (src.health <= 0 && !src.will_erase) {
                    src.will_erase = 1;
                    c.h->reward += ENEMY_REWARD;
                    int di = E::spawn_child(c, si, DUST_CLOUD, c.ents[si].rx);
                    Entity &ent = c.ents[di];
                    ent.vrot = PI_F / 0.3f;
                    ent.grow_rate = 1.0f / 1.2f;
                    ent.expire_time = 4;
                    ent.alpha_decay = 0.9f;
                    E::choose_step_random_theme(c, ent);
                }
            }
        } else if (target.type == ENEMY_BALL) {
            if (src.type == LAVA_WALL)
                target.will_erase = 1;
        }
    }
    // dodgeball.cpp:157-164
    static PG_HD void add_room(Ctx &c, float x, float y, float w, float h) {
        DodgeballState &s = st(c);
        if ((w >= s.min_dim || h >= s.min_dim) && (w >= s.hard_min_dim) && (h >= s.hard_min_dim)) {
            if (s.n_rooms >= MAX_ROOMS) {
                c.h->err |= ERR_SCRATCH_OVERFLOW;
                return;
            }
            float *r = room(c, s.n_rooms++);
            r[0] = x;
            r[1] = y;
            r[2] = w;
            r[3] = h;
        }
    }
    // dodgeball.cpp:166-224
    static PG_HD void split_room(Ctx &c, float rx, float ry, float rw, float rh, float thickness) {
        DodgeballState &s = st(c);
        MT19937 &rg = *c.rng;
        bool will_split_width = rand_rand01(rg) < .5;
        bool choice2 = rand_rand01(rg) < .5;
        if (rw < s.min_dim)
            will_split_width = false;
        if (rh < s.min_dim)
            will_split_width = true;
        float gap = (float)(.25 * (rand_randn(rg, 3) + 1));
        float pct = 1 - gap;
        if (!will_split_width) {
            float wy, wh, remy;
            if (choice2) {
                wy = ry;
                remy = ry + pct * rh;
                wh = pct * rh;
            } else {
                wy = ry + (1 - pct) * rh;
                remy = ry;
                wh = pct * rh;
            }
            int wi = E::add_entity_rxy(c, rx + rw / 2, wy + wh / 2, 0, 0, thickness, wh / 2, LAVA_WALL);
            (void)wi;
            float nextw = rw / 2 - thickness;
            add_room(c, rx, wy, nextw, wh);
            add_room(c, rx + rw / 2 + thickness, wy, nextw, wh);
            add_room(c, rx, remy, rw, rh - wh);
        } else {
            float wx, ww, remx;
            if (choice2) {
                wx = rx;
                remx = rx + pct * rw;
                ww = pct * rw;
            } else {
                wx = rx + (1 - pct) * rw;
                remx = rx;
                ww = pct * rw;
            }
            E::add_entity_rxy(c, wx + ww / 2, ry + rh / 2, 0, 0, ww / 2, thickness, LAVA_WALL);
            float nexth = rh / 2 - thickness;
            add_room(c, wx, ry, ww, nexth);
            add_room(c, wx, ry + rh / 2 + thickness, ww, nexth);
            add_room(c, remx, ry, rw - ww, rh);
        }
    }
    // dodgeball.cpp:226-238
    static PG_HD void choose_vel(Ctx &c, Entity &ent) {
        MT19937 &rg = *c.rng;
        float vel = ENEMY_VEL * (rand_randn(rg, 2) * 2 - 1);
        if (rand_randn(rg, 2) == 0) {
            ent.vx = vel;
            ent.vy = 0;
        } else {
            ent.vy = vel;
            ent.vx = 0;
        }
        ent.spawn_time = rand_randn(rg, 50) + 25;
    }
    // dodgeball.cpp:240-246
    static PG_HD float get_tile_aspect_ratio(Ctx &c, int ei) {
        const Entity &e = c.ents[ei];
        if (e.type == LAVA_WALL)
            return e.rx > e.ry ? 1 : -1;
        return 0;
    }
    // dodgeball.cpp:248-257
    static PG_HD void choose_world_dim(Ctx &c) {
        int world_dim = c.h->options.distribution_mode == MemoryMode ? 40 : 20;
        c.h->main_width = world_dim;
        c.h->main_height = world_dim;
    }
    // dodgeball.cpp:259-363
    static PG_HD void game_reset(Ctx &c) {
        E::basic_game_reset(c);
        EnvHdr &h = *c.h;
        DodgeballState &s = st(c);
        MT19937 &rg = *c.rng;
        const int mode = h.options.distribution_mode;
        h.options.center_agent = mode == MemoryMode;
        s.last_fire_time = 0;
        s.n_rooms = 0;
        {
            float *r = room(c, s.n_rooms++);
            r[0] = 0;
            r[1] = 0;
            r[2] = (float)h.main_width;
            r[3] = (float)h.main_height;
        }
        float thickness = 0.3f;
        float enemy_r = .5;
        float exit_r = .75;
        s.ball_r = .25;
        s.ball_vscale = .25;
        int num_iterations = 0;
        int max_extra_enemies = 3;
        Entity &a = agent_of(c);
        if (mode == EasyMode) {
            num_iterations = 2;
            thickness *= 2;
            enemy_r *= 2;
            s.ball_r *= 2;
            s.ball_vscale *= 2;
            h.maxspeed = .75;
            a.rx = 1;
            a.ry = 1;
            exit_r *= 2;
        } else if (mode == HardMode || mode == MemoryMode) {
            num_iterations = mode == HardMode ? 4 : 16;
            thickness = (float)(thickness * 1.5);
            enemy_r = (float)(enemy_r * 1.5);
            s.ball_r = (float)(s.ball_r * 1.5);
            s.ball_vscale = (float)(s.ball_vscale * 1.5);
            h.maxspeed = .5;
            a.rx = .75;
            a.ry = .75;
            if (mode == MemoryMode)
                max_extra_enemies = 16;
        } else if (mode == ExtremeMode) {
            num_iterations = 8;
            h.maxspeed = .25;
        } else {
            h.err |= ERR_FASSERT;
        }
        s.hard_min_dim = (float)((double)(4 * a.rx + 2 * thickness) + .5);
        s.min_dim = (float)((double)(a.rx * 8) + .5);
        for (int iteration = 0; iteration < num_iterations; iteration++) {
            if (s.n_rooms == 0)
                break;
            int idx = rand_randn(rg, s.n_rooms);
            float *r = room(c, idx);
            float rx = r[0], ry = r[1], rw = r[2], rh = r[3];
            for (int k = 4 * idx; k < 4 * (s.n_rooms - 1); k++) c.scratch[k] = c.scratch[k + 4];
            s.n_rooms--;
            split_room(c, rx, ry, rw, rh, thickness);
        }
        float border_r = 0;
        float doorlen = 2 * exit_r;
        int exit_wall_choice = rand_randn(rg, 4);
        if (exit_wall_choice == 0) {
            E::spawn_entity_rxy(c, doorlen / 2, exit_r, DOOR, 2 * border_r, 2 * border_r, h.main_width - 4 * border_r, 2 * exit_r);
        } else if (exit_wall_choice == 1) {
            E::spawn_entity_rxy(c, doorlen / 2, exit_r, DOOR, 2 * border_r, h.main_height - 2 * border_r - 2 * exit_r, h.main_width - 4 * border_r, 2 * exit_r);
        } else if (exit_wall_choice == 2) {
            E::spawn_entity_rxy(c, exit_r, doorlen / 2, DOOR, 2 * border_r, 2 * border_r, 2 * exit_r, h.main_height - 4 * border_r);
        } else if (exit_wall_choice == 3) {
            E::spawn_entity_rxy(c, exit_r, doorlen / 2, DOOR, h.main_width - 2 * border_r - 2 * exit_r, 2 * border_r, 2 * exit_r, h.main_height - 4 * border_r);
        }
        E::reposition_agent(c);
        s.num_enemies = rand_randn(rg, max_extra_enemies + 1) + 3;
        E::spawn_entities(c, s.num_enemies, enemy_r, ENEMY, 0, 0, (float)h.main_width, (float)h.main_height);
        int enemy_theme = rand_randn(rg, NUM_ENEMY_THEMES);
        for (int i = 0; i < h.n_ents; i++) {
            Entity &ent = c.ents[i];
            if (ent.type == ENEMY) {
                ent.image_theme = enemy_theme;
                ent.health = 1;
                ent.spawn_time = 0;
                ent.fire_time = 10;
                ent.collides_with_entities = 1;
                ent.smart_step = 1;
                choose_vel(c, ent);
                entity_face_direction(ent, ent.vx, ent.vy);
            } else if (ent.type == LAVA_WALL) {
                ent.collides_with_entities = 1;
            }
        }
        entity_face_direction(agent_of(c), 1, 0);
    }
    // dodgeball.cpp:365-370
    static PG_HD void fire_ball(Ctx &c, int ei, float vx, float vy) {
        DodgeballState &s = st(c);
        float ex = c.ents[ei].x, ey = c.ents[ei].y;
        int bi = E::add_entity(c, ex, ey, vx * s.ball_vscale, vy * s.ball_vscale, s.ball_r, ENEMY_BALL);
        c.ents[ei].fire_time = c.h->cur_time + rand_randn(*c.rng, 4);
        c.ents[bi].vrot = BALL_V_ROT;
        c.ents[bi].expire_time = 50;
    }
    // dodgeball.cpp:372-440
    static PG_HD void game_step(Ctx &c) {
        E::basic_game_step(c);
        EnvHdr &h = *c.h;
        DodgeballState &s = st(c);
        float vx = (float)(h.last_move_action / 3 - 1);
        float vy = (float)(h.last_move_action % 3 - 1);
        entity_face_direction(agent_of(c), vx, vy);
        if (h.special_action == 1 && (h.cur_time - s.last_fire_time) >= 7) {
            float ax = agent_of(c).x, ay = agent_of(c).y;
            int bi = E::add_entity(c, ax, ay, vx * s.ball_vscale, vy * s.ball_vscale, s.ball_r, PLAYER_BALL);
            c.ents[bi].collides_with_entities = 1;
            c.ents[bi].expire_time = 50;
            c.ents[bi].vrot = BALL_V_ROT;
            s.last_fire_time = h.cur_time;
        }
        s.num_enemies = 0;
        for (int i = h.n_ents - 1; i >= 0; i--) {
            Entity &ent = c.ents[i];
            if (ent.type == ENEMY) {
                s.num_enemies++;
                if (ent.spawn_time == 0)
                    choose_vel(c, ent);
                else
                    ent.spawn_time -= 1;
                bool can_fire = (h.cur_time - ent.fire_time) >= s.enemy_fire_delay;
                if (can_fire) {
                    const Entity &a = agent_of(c);
                    float dx = ent.x - a.x;
                    float dy = ent.y - a.y;
                    float bvelx = (ent.x < a.x ? 1 : -1);
                    float bvely = (ent.y < a.y ? 1 : -1);
                    if (pg_dfabs((double)dx) < 1) {
                        fire_ball(c, i, 0, bvely);
                        c.ents[i].vx = 0;
                        c.ents[i].vy = bvely * ENEMY_VEL;
                    } else if (pg_dfabs((double)dy) < 1) {
                        fire_ball(c, i, bvelx, 0);
                        c.ents[i].vx = bvelx * ENEMY_VEL;
                        c.ents[i].vy = 0;
                    }
                }
                entity_face_direction(c.ents[i], c.ents[i].vx, c.ents[i].vy);
            } else if (ent.type == PLAYER_BALL || ent.type == ENEMY_BALL) {
                if (ent.x < ent.rx || ent.x > (h.main_width - ent.rx))
                    ent.will_erase = 1;
                else if (ent.y < ent.ry || ent.y > (h.main_height - ent.ry))
                    ent.will_erase = 1;
            }
        }
        E::erase_if_needed(c);
    }
};

}  // namespace pg
