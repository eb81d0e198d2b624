// Chaser on the device engine. Behaviour restated from games/chaser.cpp (cited per function).
#pragma once
#include "../pg_mazegen.cuh"
#include "../pg_raster.cuh"

namespace pg {

struct ChaserState {
    int32_t eat_timeout, egg_timeout, eat_time, total_enemies, total_orbs, orbs_collected, maze_dim;
    int32_t n_free_cells;
};

struct ChaserGame : Defaults<ChaserGame>, DrawDefaults<ChaserGame> {
    using E = Engine<ChaserGame>;
    static constexpr int ENT_CAP = 32;
    static constexpr int GRID_CAP = 19 * 19;
    static constexpr int MAZE_WORDS = 4800;       // MazeGen::words_needed(19) = 4721
    static constexpr int LIST_WORDS = 400;
    static constexpr int SCRATCH_WORDS = MAZE_WORDS + 4 * LIST_WORDS;
    static constexpr int PERSIST_SCRATCH_FIRST = MAZE_WORDS;  // free_cells and is_space_vec; the maze and the quadrant lists are workspace
    static constexpr int PERSIST_SCRATCH_WORDS = 2 * LIST_WORDS;
    static constexpr int MAX_VISIBLE_ENTS = 64;
    static constexpr int MAX_ROT_BLITS = 0;
    static constexpr int MAX_VIEW_CELLS = 19;
    static constexpr const char *NAME = "chaser";
    // superset of the types is_blocked accepts; nothing reflects
    static PG_HD bool may_be_obstacle(Ctx &c, int t) { return t == WALL_OBJ || t == c.oob || t == MAZE_WALL; }
    static PG_HD bool may_block_or_reflect(Ctx &c, int src, int t) { return may_be_obstacle(c, t); }

    // chaser.cpp:10-23
    static constexpr float ORB_REWARD = 0.04f;
    static constexpr float COMPLETION_BONUS = 10.0f;
    static constexpr float ORB_DIM = 0.3f;
    static constexpr int LARGE_ORB = 2, ENEMY_WEAK = 3, ENEMY_EGG = 4, MAZE_WALL = 5, ENEMY = 6, ENEMY2 = 7, ENEMY3 = 8;
    static constexpr int MARKER = 1001, ORB = 1002;

    static PG_HD ChaserState &st(Ctx &c) { return game_state<ChaserState>(c); }
    static PG_HD int32_t *free_cells(Ctx &c) { return c.scratch + MAZE_WORDS; }
    static PG_HD int32_t *is_space_vec(Ctx &c) { return c.scratch + MAZE_WORDS + LIST_WORDS; }

    // chaser.cpp:39-49
    static PG_HD void init_constants(Ctx &c) {
        base_init_constants(c);
        c.h->mixrate = 1;
        c.h->maxspeed = .5;
        st(c).eat_timeout = 75;
        st(c).egg_timeout = 50;
        c.h->has_useful_vel_info = 0;
    }
    // chaser.cpp:81-90
    static PG_HD void update_agent_velocity(Ctx &c) {
        EnvHdr &h = *c.h;
        Entity &a = agent_of(c);
        if (h.action_vx != 0)
            a.vx = h.maxspeed * h.action_vx;
        if (h.action_vy != 0)
            a.vy = h.maxspeed * h.action_vy;
        a.vx = (float)(pg_sign((double)a.vx) * (double)h.maxspeed);
        a.vy = (float)(pg_sign((double)a.vy) * (double)h.maxspeed);
    }
    // chaser.cpp:92-97
    static PG_HD bool is_blocked(Ctx &c, int src, int target, bool is_horizontal) {
        if (target == MAZE_WALL)
            return true;
        return Defaults<ChaserGame>::is_blocked(c, src, target, is_horizontal);
    }
    static PG_HD bool can_eat_enemies(Ctx &c) { return c.h->cur_time - st(c).eat_time < st(c).eat_timeout; }
    // chaser.cpp:99-112
    static PG_HD int image_for_type(Ctx &c, int type) {
        if (type == ENEMY) {
            if (can_eat_enemies(c))
                return ENEMY_WEAK;
            int rem = (c.h->cur_time / 2) % 4;
            if (rem == 3)
                rem = 1;
            return ENEMY + rem;
        }
        return Defaults<ChaserGame>::image_for_type(c, type);
    }
    // chaser.cpp:114-120: ORB cells are a green square, 30 % of the cell, centred
    template <class Frame>
    static PG_HD bool make_grid_obj_blit(Ctx &c, const Frame &f, Blit &b, double *rect, int type, int theme) {
        if (type != ORB)
            return DrawDefaults<ChaserGame>::make_grid_obj_blit(c, f, b, rect, type, theme);
        double x = rect[0] + rect[2] * (double)(1 - ORB_DIM) / 2;
        double y = rect[1] + rect[3] * (double)(1 - ORB_DIM) / 2;
        make_solid_blit(b, x, y, rect[2] * (double)ORB_DIM, rect[3] * (double)ORB_DIM, (0u << 16) | (255u << 8) | 0u);
        return true;
    }
    // chaser.cpp:122-138
    static PG_HD void handle_agent_collision(Ctx &c, int oi) {
        Entity &obj = c.ents[oi];
        if (obj.type == LARGE_ORB) {
            st(c).eat_time = c.h->cur_time;
            c.h->reward += ORB_REWARD;
            obj.will_erase = 1;
        } else if (obj.type == ENEMY) {
            if (can_eat_enemies(c))
                obj.will_erase = 1;
            else
                c.h->done = 1;
        }
    }
    // chaser.cpp:140-143
    static PG_HD void choose_world_dim(Ctx &c) {
        c.h->main_width = st(c).maze_dim;
        c.h->main_height = st(c).maze_dim;
    }
    // chaser.cpp:287-290
    static PG_HD void spawn_egg(Ctx &c, int enemy_cell) {
        const int md = st(c).maze_dim;
        int ei = E::add_entity(c, (float)((enemy_cell % md) + .5), (float)((enemy_cell / md) + .5), 0, 0, .5, ENEMY_EGG);
        c.ents[ei].health = (float)st(c).egg_timeout;
    }
    // RandGen::simple_choose, randgen.cpp:72-93 (rejection against a set; flags live in scratch)
    static PG_HD void simple_choose(Ctx &c, int n, int k, int32_t *chosen, int32_t *flags) {
        pg_warp_for(n, [=](int i) { flags[i] = 0; });
        for (int i = 0; i < k; i++) {
            int next = rand_randn(*c.rng, n);
            while (flags[next]) next = rand_randn(*c.rng, n);
            chosen[i] = next;
            flags[next] = 1;
        }
    }

    // chaser.cpp:145-281
    static PG_HD void game_reset(Ctx &c) {
        EnvHdr &h = *c.h;
        ChaserState &s = st(c);
        int extra_orb_sign = 1;
        if (h.options.distribution_mode == EasyMode) {
            s.maze_dim = 11;
            s.total_enemies = 3;
            extra_orb_sign = 0;
        } else if (h.options.distribution_mode == HardMode) {
            s.maze_dim = 13;
            s.total_enemies = 3;
            extra_orb_sign = -1;
        } else if (h.options.distribution_mode == ExtremeMode) {
            s.maze_dim = 19;
            s.total_enemies = 5;
            extra_orb_sign = 1;
        }
        const int maze_dim = s.maze_dim;
        E::basic_game_reset(c);
        h.options.center_agent = 0;
        agent_of(c).rx = .5;
        agent_of(c).ry = .5;
        s.eat_time = -1 * s.eat_timeout;
        E::fill_elem(c, 0, 0, h.main_width, h.main_height, MAZE_WALL);
        MazeGen mg;
        mg.init(c, maze_dim);
        mg.generate_maze_no_dead_ends();

        int32_t *fc = free_cells(c);
        int32_t *quad = c.scratch + MAZE_WORDS + 2 * LIST_WORDS;  // 4 quadrant lists of <= 100 each
        int32_t *flags = c.scratch + MAZE_WORDS + 3 * LIST_WORDS;
        int nquad[4] = {0, 0, 0, 0};
        int orbs_for_quadrant[4];
        const int num_quadrants = 4;
        int extra_quad = rand_randn(*c.rng, num_quadrants);
        for (int i = 0; i < num_quadrants; i++) orbs_for_quadrant[i] = 1 + (i == extra_quad ? extra_orb_sign : 0);
        for (int i = 0; i < maze_dim; i++) {
            for (int j = 0; j < maze_dim; j++) {
                int obj = mg.grid_get(i + MAZE_OFFSET, j + MAZE_OFFSET);
                E::set_obj(c, i, j, obj == WALL_OBJ ? MAZE_WALL : obj);
                if (obj == SPACE) {
                    int idx = j * maze_dim + i;
                    int quad_idx = (i >= maze_dim / 2.0 ? 1 : 0) * 2 + (j >= maze_dim / 2.0 ? 1 : 0);
                    if (nquad[quad_idx] < 100)
                        quad[quad_idx * 100 + nquad[quad_idx]++] = idx;
                    else
                        h.err |= ERR_SCRATCH_OVERFLOW;
                }
            }
        }
        for (int i = 0; i < num_quadrants; i++) {
            int num_orbs = orbs_for_quadrant[i];
            int sel[4];
            simple_choose(c, nquad[i], num_orbs, sel, flags);
            for (int q = 0; q < num_orbs; q++) {
                int cell = quad[i * 100 + sel[q]];
                E::spawn_entity_at_idx(c, cell, 0.4f, LARGE_ORB);
                E::set_obj_idx(c, cell, MARKER);
            }
        }
        int nfree = 0;
        for (int i = 0; i < h.grid_size; i++)
            if (c.grid[i] == SPACE)
                fc[nfree++] = i;
        int sel[8];
        simple_choose(c, nfree, 1 + s.total_enemies, sel, flags);
        int start = fc[sel[0]];
        agent_of(c).x = (float)((start % maze_dim) + .5);
        agent_of(c).y = (float)((start / maze_dim) + .5);
        for (int i = 0; i < s.total_enemies; i++) {
            int cell = fc[sel[i + 1]];
            E::set_obj_idx(c, cell, MARKER);
            spawn_egg(c, cell);
        }
        for (int q = 0; q < nfree; q++) E::set_obj_idx(c, fc[q], ORB);
        s.total_orbs = nfree;
        s.orbs_collected = 0;
        for (int i = 0; i < h.grid_size; i++)
            if (c.grid[i] == MARKER)
                c.grid[i] = (int16_t)SPACE;
        int32_t *isv = is_space_vec(c);
        nfree = 0;
        for (int i = 0; i < h.grid_size; i++) {
            bool is_space = E::get_obj_idx(c, i) != MAZE_WALL;
            if (is_space)
                fc[nfree++] = i;
            isv[i] = is_space;
        }
        s.n_free_cells = nfree;
    }

    static PG_HD int manhattan_dist(Ctx &c, int a, int b) {
        const int w = c.h->main_width;
        int dx = (a % w) - (b % w), dy = (a / w) - (b / w);
        return (dx < 0 ? -dx : dx) + (dy < 0 ? -dy : dy);
    }

    // chaser.cpp:316-397
    static PG_HD void game_step(Ctx &c) {
        E::basic_game_step(c);
        EnvHdr &h = *c.h;
        ChaserState &s = st(c);
        int num_enemies = 0;
        float default_enemy_speed = .5;
        float vscale = can_eat_enemies(c) ? (float)(default_enemy_speed * .5) : default_enemy_speed;
        const int32_t *isv = is_space_vec(c);
        for (int j = h.n_ents - 1; j >= 0; j--) {
            Entity &ent = c.ents[j];
            if (ent.type == ENEMY_EGG) {
                num_enemies++;
                ent.health -= 1;
                if (ent.health == 0) {
                    ent.will_erase = 1;
                    int ci = E::spawn_child(c, j, ENEMY, .5);
                    c.ents[ci].smart_step = 1;
                }
            } else if (ent.type == ENEMY) {
                num_enemies++;
                float x = (float)(ent.x - .5);
                float y = (float)(ent.y - .5);
                int dist_scale = can_eat_enemies(c) ? -1 : 1;
                int enemy_idx = E::to_grid_idx(c, (int)x, (int)y);
                int agent_idx = E::to_grid_idx(c, (int)agent_of(c).x, (int)agent_of(c).y);
                bool is_at_junction = pg_dfabs((double)x - round((double)x)) + pg_dfabs((double)y - round((double)y)) < .01;
                bool be_agressive = h.step_rand_int % 2 == 0;
                if ((ent.vx == 0 && ent.vy == 0) || is_at_junction) {
                    int space_neighbors[4];
                    int nsn = 0;
                    int prev_idx = E::to_grid_idx(c, (int)((double)x - pg_sign((double)ent.vx)), (int)((double)y - pg_sign((double)ent.vy)));
                    const int ex = enemy_idx % h.main_width, ey = enemy_idx / h.main_width;
                    int min_dist = 2 * h.main_width;
                    for (int di = -1; di <= 1; di++) {
                        for (int dj = -1; dj <= 1; dj++) {
                            if (di == 0 && dj == 0)
                                continue;
                            if (di != 0 && dj != 0)
                                continue;
                            int adj = E::to_grid_idx(c, ex + di, ey + dj);
                            if (adj == INVALID_IDX)
                                continue;
                            if (isv[adj] && adj != prev_idx) {
                                int md = manhattan_dist(c, adj, agent_idx) * dist_scale;
                                if (be_agressive) {
                                    if (md < min_dist) {
                                        min_dist = md;
                                        nsn = 0;
                                        space_neighbors[nsn++] = adj;
                                    } else if (md == min_dist) {
                                        space_neighbors[nsn++] = adj;
                                    }
                                } else {
                                    space_neighbors[nsn++] = adj;
                                }
                            }
                        }
                    }
                    if (nsn == 0) {
                        h.err |= ERR_FASSERT;  // reference: modulo by zero
                        continue;
                    }
                    int neighbor = space_neighbors[h.step_rand_int % nsn];
                    int nx = neighbor % h.main_width;
                    int ny = neighbor / h.main_width;
                    ent.vx = (nx - x) * vscale;
                    ent.vy = (ny - y) * vscale;
                }
            }
        }
        if (num_enemies < s.total_enemies) {
            int selected_idx = h.step_rand_int % s.n_free_cells;
            spawn_egg(c, free_cells(c)[selected_idx]);
        }
        int agent_idx = E::get_agent_index(c);
        if (E::get_obj_idx(c, agent_idx) == ORB) {
            E::set_obj_idx(c, agent_idx, SPACE);
            h.reward += ORB_REWARD;
            s.orbs_collected += 1;
        }
        if (s.orbs_collected == s.total_orbs) {
            h.reward += COMPLETION_BONUS;
            h.level_complete = 1;
            h.done = 1;
        }
    }
};

}  // namespace pg
