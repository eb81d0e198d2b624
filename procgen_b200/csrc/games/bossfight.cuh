// BossFight on the device engine. Behaviour restated from games/bossfight.cpp (cited per function).
#pragma once
#include "../pg_raster.cuh"

namespace pg {

struct BossfightState {
    int32_t boss_idx, shields_idx;  // the reference holds shared_ptrs; indices are kept in step by on_entity_moved
    int32_t attack_modes[8];
    int32_t n_attack_modes;
    int32_t last_fire_time, time_to_swap, invulnerable_duration, vulnerable_duration, num_rounds, round_num, round_health;
    int32_t boss_vel_timeout, curr_vel_timeout, attack_mode, player_laser_theme, boss_laser_theme, damaged_until_time;
    int32_t shields_are_up, barriers_moves_right;
    float base_fire_prob, boss_bullet_vel, barrier_vel, barrier_spawn_prob, rand_pct, rand_fire_pct, rand_pct_x, rand_pct_y;
};

struct BossfightGame : Defaults<BossfightGame>, DrawDefaults<BossfightGame> {
    using E = Engine<BossfightGame>;
    static constexpr int ENT_CAP = 384;
    static constexpr int GRID_CAP = 20 * 20;
    static constexpr int SCRATCH_WORDS = 0;
    // rand_pct, rand_fire_pct, rand_pct_x, rand_pct_y: drawn at the start of every step, never by game_reset
    static constexpr int STEP_STATE_OFFSET = (int)offsetof(BossfightState, rand_pct);
    static constexpr int STEP_STATE_BYTES = 4 * (int)sizeof(float);
    static constexpr int MAX_VISIBLE_ENTS = 384;
    static constexpr int MAX_ROT_BLITS = 352;  // every enemy bullet and its trails spin (vrot = PI/8)
    static constexpr int MAX_VIEW_CELLS = 20;
    static constexpr const char *NAME = "bossfight";
    static constexpr bool DRAWS_GRID = false;  // entities only; the grid stays all SPACE
    // is_blocked / is_blocked_ents / will_reflect are the engine defaults here: only an entity typed WALL_OBJ or as the out-of-bounds object could block
    static PG_HD bool may_be_obstacle(Ctx &c, int t) { return t == WALL_OBJ || t == c.oob; }
    static PG_HD bool may_block_or_reflect(Ctx &c, int src, int t) { return may_be_obstacle(c, t); }

    // bossfight.cpp:8-30
    static constexpr int COMPLETION_BONUS = 10, POSITIVE_REWARD = 1;
    static constexpr int PLAYER_BULLET = 1, BOSS = 2, SHIELDS = 3, ENEMY_BULLET = 4, LASER_TRAIL = 5, REFLECTED_BULLET = 6, BARRIER = 7;
    static constexpr float BOSS_R = 3;
    static constexpr int NUM_ATTACK_MODES = 4, NUM_LASER_THEMES = 3, PLAYER_BULLET_VEL = 1, BOTTOM_MARGIN = 6;
    static constexpr int BOSS_VEL_TIMEOUT = 20, BOSS_DAMAGED_TIMEOUT = 40;

    static PG_HD BossfightState &st(Ctx &c) { return game_state<BossfightState>(c); }
    static PG_HD Entity &boss(Ctx &c) { return c.ents[st(c).boss_idx]; }
    static PG_HD Entity &shields(Ctx &c) { return c.ents[st(c).shields_idx]; }

    static constexpr bool HAS_ENTITY_HOOKS = true;
    static PG_HD void on_entity_moved(Ctx &c, int from, int to) {
        BossfightState &s = st(c);
        if (s.boss_idx == from)
            s.boss_idx = to;
        if (s.shields_idx == from)
            s.shields_idx = to;
    }

    // bossfight.cpp:62-71
    static PG_HD void init_constants(Ctx &c) {
        base_init_constants(c);
        c.h->timeout = 4000;
        c.h->main_width = 20;
        c.h->main_height = 20;
        c.h->mixrate = .5;
        c.h->maxspeed = 0.85f;
    }
    // bossfight.cpp:111-122
    static PG_HD void handle_agent_collision(Ctx &c, int oi) {
        int t = c.ents[oi].type;
        if (t == BOSS || t == BARRIER || t == ENEMY_BULLET)
            c.h->done = 1;
    }
    // bossfight.cpp:124-129
    static PG_HD bool should_draw_entity(Ctx &c, int ei) {
        if (c.ents[ei].type == SHIELDS)
            return st(c).shields_are_up != 0;
        return true;
    }
    // bossfight.cpp:198-205
    static PG_HD void prepare_boss(Ctx &c) {
        BossfightState &s = st(c);
        s.shields_are_up = 1;
        s.curr_vel_timeout = s.boss_vel_timeout;
        s.time_to_swap = s.invulnerable_duration;
        s.attack_mode = s.attack_modes[s.round_num % s.n_attack_modes];
        boss(c).vx = 0;
        boss(c).vy = 0;
    }
    // bossfight.cpp:131-196
    static PG_HD void handle_collision(Ctx &c, int si, int ti) {
        EnvHdr &h = *c.h;
        BossfightState &s = st(c);
        if (c.ents[si].type == PLAYER_BULLET) {
            bool will_erase = false;
            Entity &src = c.ents[si];
            Entity &target = c.ents[ti];
            if (target.type == SHIELDS) {
                if (s.shields_are_up) {
                    src.type = REFLECTED_BULLET;
                    float theta = (float)((double)PI_F * (1.25 + .5 * (double)s.rand_pct));
                    src.vy = (float)(PLAYER_BULLET_VEL * sin((double)theta) * .5);
                    src.vx = (float)(PLAYER_BULLET_VEL * cos((double)theta) * .5);
                    src.expire_time = 4;
                    src.life_time = 0;
                    src.alpha_decay = 0.8f;
                }
            } else if (target.type == BOSS) {
                if (!s.shields_are_up) {
                    target.health -= 1;
                    will_erase = true;
                    if (int(target.health) % s.round_health == 0) {
                        h.reward += POSITIVE_REWARD;
                        if (target.health == 0) {
                            h.done = 1;
                            h.reward += COMPLETION_BONUS;
                            h.level_complete = 1;
                        } else {
                            s.round_num++;
                            prepare_boss(c);
                            s.curr_vel_timeout = BOSS_DAMAGED_TIMEOUT;
                            s.damaged_until_time = h.cur_time + BOSS_DAMAGED_TIMEOUT;
                        }
                    }
                }
            }
            if (will_erase && !c.ents[si].will_erase) {
                c.ents[si].will_erase = 1;
                int xi = E::spawn_child(c, si, EXPLOSION, (float)(.5 * c.ents[si].rx));
                c.ents[xi].vx = c.ents[ti].vx;
                c.ents[xi].vy = c.ents[ti].vy;
            }
        } else if (c.ents[si].type == BARRIER) {
            int tt = c.ents[ti].type;
            if (tt == ENEMY_BULLET || tt == PLAYER_BULLET) {
                c.ents[ti].will_erase = 1;
                E::spawn_child(c, ti, EXPLOSION, (float)(.5 * c.ents[ti].rx));
            } else if (tt == LASER_TRAIL) {
                c.ents[ti].will_erase = 1;
            }
            if (c.ents[si].health <= 0) {
                if (!c.ents[si].will_erase) {
                    int xi = E::spawn_child(c, si, EXPLOSION, (float)(.5 * c.ents[si].rx));
                    c.ents[xi].vx = c.ents[si].vx;
                    c.ents[xi].vy = c.ents[si].vy;
                }
                c.ents[si].will_erase = 1;
            }
        }
    }
    // bossfight.cpp:336-354
    static PG_HD void spawn_barriers(Ctx &c) {
        EnvHdr &h = *c.h;
        MT19937 &rg = *c.rng;
        int num_barriers = rand_randn(rg, 3) + 1;
        for (int i = 0; i < num_barriers; i++) {
            float barrier_r = 0.6f;
            float min_barrier_y = (float)((double)(2 * agent_of(c).ry + barrier_r) + .5);
            float ent_y = rand_rand01(rg) * (BOTTOM_MARGIN - min_barrier_y - barrier_r) + min_barrier_y;
            float ent_x = rand_rand01(rg) * (h.main_width - 2 * barrier_r) + barrier_r;
            if (h.n_ents >= c.ent_cap) {
                h.err |= ERR_ENTITY_OVERFLOW;
                continue;
            }
            Entity &ent = c.ents[h.n_ents];
            entity_init(ent, ent_x, ent_y, 0, 0, barrier_r, barrier_r, BARRIER);
            E::choose_random_theme(c, ent);
            E::match_aspect_ratio(c, ent);
            ent.health = 3;
            ent.collides_with_entities = 1;
            if (!E::has_any_collision(c, ent))
                E::push_entity(c);
        }
    }
    // bossfight.cpp:207-264
    static PG_HD void game_reset(Ctx &c) {
        E::basic_game_reset(c);
        EnvHdr &h = *c.h;
        BossfightState &s = st(c);
        MT19937 &rg = *c.rng;
        s.damaged_until_time = 0;
        s.last_fire_time = 0;
        s.boss_bullet_vel = h.options.distribution_mode == EasyMode ? .5 : .75;
        int max_extra_invulnerable = h.options.distribution_mode == EasyMode ? 1 : 3;
        h.options.center_agent = 0;
        s.boss_idx = E::add_entity(c, (float)(h.main_width / 2), (float)(h.main_height / 2), 0, 0, BOSS_R, BOSS);
        E::choose_random_theme(c, boss(c));
        E::match_aspect_ratio(c, boss(c));
        {
            float bx = boss(c).x, by = boss(c).y, brx = (float)(1.2 * boss(c).rx), bry = (float)(1.2 * boss(c).ry);
            s.shields_idx = E::add_entity_rxy(c, bx, by, 0, 0, brx, bry, SHIELDS);
        }
        s.boss_vel_timeout = BOSS_VEL_TIMEOUT;
        s.base_fire_prob = 0.1f;
        s.round_health = rand_randn(rg, 9) + 1;
        s.num_rounds = 1 + rand_randn(rg, 5);
        s.invulnerable_duration = 2 + rand_randn(rg, max_extra_invulnerable + 1);
        s.vulnerable_duration = 500;
        boss(c).health = (float)(s.round_health * s.num_rounds);
        E::choose_random_theme(c, agent_of(c));
        s.player_laser_theme = rand_randn(rg, NUM_LASER_THEMES);
        s.boss_laser_theme = rand_randn(rg, NUM_LASER_THEMES);
        s.n_attack_modes = 0;
        for (int i = 0; i < s.num_rounds; i++) s.attack_modes[s.n_attack_modes++] = rand_randn(rg, NUM_ATTACK_MODES);
        s.round_num = 0;
        prepare_boss(c);
        Entity &a = agent_of(c);
        a.rx = .75;
        E::match_aspect_ratio(c, a);
        E::reposition_agent(c);
        a.y = a.ry;
        s.barrier_vel = 0.1f;
        s.barriers_moves_right = rand_randbool(rg);
        s.barrier_spawn_prob = 0.025f;
        spawn_barriers(c);
    }
    // bossfight.cpp:266-271 — cos/sin are the double overloads
    static PG_HD void boss_fire(Ctx &c, float bullet_r, float vel, float theta) {
        float bx = boss(c).x, by = boss(c).y;
        int bi = E::add_entity(c, bx, by, (float)((double)vel * cos((double)theta)), (float)((double)vel * sin((double)theta)), bullet_r, ENEMY_BULLET);
        c.ents[bi].image_theme = st(c).boss_laser_theme;
        c.ents[bi].expire_time = 50;
        c.ents[bi].vrot = PI_F / 8;
    }
    // bossfight.cpp:273-334
    static PG_HD void active_attack(Ctx &c) {
        EnvHdr &h = *c.h;
        BossfightState &s = st(c);
        if (s.attack_mode == 0) {
            if (h.cur_time % 8 == 0)
                for (int i = 0; i < 5; i++) boss_fire(c, .5, s.boss_bullet_vel, (float)((double)PI_F * 1.5 + (double)((i - 2) * PI_F / 8)));
        } else if (s.attack_mode == 1) {
            int dt = 5;
            if (h.cur_time % dt == 0) {
                int k = h.cur_time / dt;
                k = 8 - (k % 16);
                if (k < 0)
                    k = -k;
                for (int i = 0; i < 4; i++) boss_fire(c, .5, s.boss_bullet_vel, (float)((double)PI_F * (1.25 + .5 * k / 8.0) + (double)(i * PI_F / 2)));
            }
        } else if (s.attack_mode == 2) {
            if (h.cur_time % 10 == 0) {
                int num_bullets = 8;
                float offset = s.rand_pct * 2 * PI_F;
                for (int i = 0; i < num_bullets; i++) {
                    float vel = s.boss_bullet_vel;
                    float theta = 2 * PI_F / num_bullets * i + offset;
                    boss_fire(c, .5, vel, theta);
                }
            }
        } else if (s.attack_mode == 3) {
            if (h.cur_time % 4 == 0)
                boss_fire(c, .5, s.boss_bullet_vel, PI_F * (1 + s.rand_pct));
        }
    }
    // bossfight.cpp:356-431
    static PG_HD void game_step(Ctx &c) {
        E::basic_game_step(c);
        EnvHdr &h = *c.h;
        BossfightState &s = st(c);
        MT19937 &rg = *c.rng;
        shields(c).x = boss(c).x;
        shields(c).y = boss(c).y;
        s.rand_pct = rand_rand01(rg);
        s.rand_fire_pct = rand_rand01(rg);
        s.rand_pct_x = rand_rand01(rg);
        s.rand_pct_y = rand_rand01(rg);
        if (s.curr_vel_timeout <= 0) {
            float dest_x = s.rand_pct_x * (h.main_width - 2 * BOSS_R) + BOSS_R;
            float dest_y = s.rand_pct_y * (h.main_height - 2 * BOSS_R - BOTTOM_MARGIN) + BOSS_R + BOTTOM_MARGIN;
            boss(c).vx = (dest_x - boss(c).x) / s.boss_vel_timeout;
            boss(c).vy = (dest_y - boss(c).y) / s.boss_vel_timeout;
            s.curr_vel_timeout = s.boss_vel_timeout;
            if (s.time_to_swap > 0) {
                s.time_to_swap -= 1;
            } else {
                s.time_to_swap = s.shields_are_up ? s.vulnerable_duration : s.invulnerable_duration;
                s.shields_are_up = !s.shields_are_up;
            }
        } else {
            s.curr_vel_timeout -= 1;
        }
        if (h.special_action == 1 && (h.cur_time - s.last_fire_time) >= 3) {
            float ax = agent_of(c).x, ay = agent_of(c).y;
            int bi = E::add_entity(c, ax, ay, 0, PLAYER_BULLET_VEL, .25, PLAYER_BULLET);
            c.ents[bi].image_theme = s.player_laser_theme;
            c.ents[bi].collides_with_entities = 1;
            c.ents[bi].expire_time = 25;
            s.last_fire_time = h.cur_time;
        }
        if (s.damaged_until_time >= h.cur_time) {
            if (h.cur_time % 3 == 0) {
                float pos_x = boss(c).x + (2 * s.rand_pct_x - 1) * boss(c).rx;
                float pos_y = boss(c).y + (2 * s.rand_pct_y - 1) * boss(c).ry;
                E::add_entity(c, pos_x, pos_y, 0, 0, .75, EXPLOSION);
            }
        } else if (s.shields_are_up) {
            active_attack(c);
        } else {
            if (s.rand_fire_pct < s.base_fire_prob)
                boss_fire(c, .5, s.boss_bullet_vel, PI_F * (1 + s.rand_pct));
        }
        for (int i = h.n_ents - 1; i >= 0; i--) {
            if (c.ents[i].type == ENEMY_BULLET) {
                float v_trail = .5;
                const Entity e = c.ents[i];
                int ti = E::add_entity_rxy(c, e.x, e.y, e.vx * v_trail, e.vy * v_trail, e.rx, e.ry, LASER_TRAIL);
                Entity &trail = c.ents[ti];
                trail.alpha_decay = 0.7f;
                trail.image_type = ENEMY_BULLET;
                trail.image_theme = s.boss_laser_theme;
                trail.vrot = e.vrot;
                trail.rotation = e.rotation;
                trail.expire_time = 8;
            }
        }
    }
};

}  // namespace pg
