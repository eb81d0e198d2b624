// Miner on the device engine. Behaviour restated from games/miner.cpp (cited per function).
#pragma once
#include "../pg_raster.cuh"

namespace pg {

struct MinerState {
    int32_t diamonds_remaining;
};

struct MinerGame : Defaults<MinerGame>, DrawDefaults<MinerGame> {
    using E = Engine<MinerGame>;
    static constexpr int ENT_CAP = 16;
    static constexpr int GRID_CAP = 35 * 35;
    static constexpr int SCRATCH_WORDS = 4 * 1280;
    // diamonds_remaining: counted by every step, never by game_reset
    static constexpr int STEP_STATE_OFFSET = (int)offsetof(MinerState, diamonds_remaining);
    static constexpr int STEP_STATE_BYTES = (int)sizeof(int32_t);
    static constexpr int MAX_VISIBLE_ENTS = 64;
    static constexpr int MAX_ROT_BLITS = 0;
    static constexpr bool ENTS_BELOW_GRID = true;  // the exit sits under the grid layer (render_z = -1, miner.cpp:199)
    static constexpr int MAX_VIEW_CELLS = 20;  // hard: whole 20x20 world; memory mode is centred (11)
    static constexpr const char *NAME = "miner";
    // superset of the types is_blocked and will_reflect accept
    static PG_HD bool may_be_obstacle(Ctx &c, int t) { return t == WALL_OBJ || t == c.oob || t == OOB_WALL || t == BOULDER || t == MOVING_BOULDER || t == DIAMOND || t == MOVING_DIAMOND; }
    static PG_HD bool may_block_or_reflect(Ctx &c, int src, int t) { return may_be_obstacle(c, t); }

    // miner.cpp:8-19
    static constexpr float COMPLETION_BONUS = 10.0;
    static constexpr int DIAMOND_REWARD = 1;
    static constexpr int BOULDER = 1, DIAMOND = 2, MOVING_BOULDER = 3, MOVING_DIAMOND = 4, ENEMY = 5, EXIT = 6, DIRT = 9;
    static constexpr int OOB_WALL = 10;

    static PG_HD MinerState &st(Ctx &c) { return game_state<MinerState>(c); }

    // miner.cpp:25-36
    static PG_HD void init_constants(Ctx &c) {
        base_init_constants(c);
        c.h->main_width = 20;
        c.h->main_height = 20;
        c.h->mixrate = .5;
        c.h->maxspeed = .5;
        c.h->has_useful_vel_info = 0;
        c.h->out_of_bounds_object = OOB_WALL;
        c.h->visibility = 8.0;
    }
    // miner.cpp:58-69
    static PG_HD bool is_blocked(Ctx &c, int src, int target, bool is_horizontal) {
        if (Defaults<MinerGame>::is_blocked(c, src, target, is_horizontal))
            return true;
        if (c.ents[src].type == PLAYER && (target == BOULDER || target == MOVING_BOULDER || target == OOB_WALL))
            return true;
        return false;
    }
    static PG_HD bool will_reflect(Ctx &c, int src, int target) {
        return (src == ENEMY && (target == BOULDER || target == DIAMOND || target == MOVING_BOULDER || target == MOVING_DIAMOND || target == c.oob));
    }
    // miner.cpp:71-83
    static PG_HD void handle_agent_collision(Ctx &c, int oi) {
        int t = c.ents[oi].type;
        if (t == ENEMY) {
            c.h->done = 1;
        } else if (t == EXIT) {
            if (st(c).diamonds_remaining == 0) {
                c.h->reward += COMPLETION_BONUS;
                c.h->level_complete = 1;
                c.h->done = 1;
            }
        }
    }
    // miner.cpp:85-93
    static PG_HD int image_for_type(Ctx &c, int type) {
        if (type == MOVING_BOULDER)
            return BOULDER;
        if (type == MOVING_DIAMOND)
            return DIAMOND;
        return Defaults<MinerGame>::image_for_type(c, type);
    }
    // miner.cpp:99-103
    static PG_HD void set_action_xy(Ctx &c, int move_action) {
        Defaults<MinerGame>::set_action_xy(c, move_action);
        if (c.h->action_vx != 0)
            c.h->action_vy = 0;
    }
    // miner.cpp:105-115
    static PG_HD void choose_new_vel(Ctx &c, Entity &ent) {
        int is_horizontal = rand_randbool(*c.rng);
        int vel = rand_randn(*c.rng, 2) * 2 - 1;
        if (is_horizontal) {
            ent.vx = vel;
            ent.vy = 0;
        } else {
            ent.vx = 0;
            ent.vy = vel;
        }
    }
    // miner.cpp:117-130
    static PG_HD void choose_world_dim(Ctx &c) {
        int dist_diff = c.h->options.distribution_mode;
        if (dist_diff == EasyMode) {
            c.h->main_width = 10;
            c.h->main_height = 10;
        } else if (dist_diff == HardMode) {
            c.h->main_width = 20;
            c.h->main_height = 20;
        } else if (dist_diff == MemoryMode) {
            c.h->main_width = 35;
            c.h->main_height = 35;
        }
    }
    // miner.cpp:132-199; RandGen::simple_choose randgen.cpp:72-93 (rejection against a set)
    static PG_HD void game_reset(Ctx &c) {
        E::basic_game_reset(c);
        EnvHdr &h = *c.h;
        Entity &a = agent_of(c);
        a.rx = .5;
        a.ry = .5;
        const int main_area = h.main_height * h.main_width;
        h.options.center_agent = h.options.distribution_mode == MemoryMode;
        h.grid_step = 1;
        float diamond_pct = 12 / 400.0f;
        float boulder_pct = 80 / 400.0f;
        int num_diamonds = (int)(diamond_pct * h.grid_size);
        int num_boulders = (int)(boulder_pct * h.grid_size);
        const int k = num_diamonds + num_boulders + 1;
        int32_t *flag = c.scratch;            // [main_area]
        int32_t *obj_idxs = c.scratch + 1280; // [k]
        int32_t *dirt_cells = c.scratch + 2 * 1280;
        int32_t *cands = c.scratch + 3 * 1280;
        if (main_area > 1280 || k > 1280) {
            h.err |= ERR_SCRATCH_OVERFLOW;
            return;
        }
        pg_warp_for(main_area, [=](int i) { flag[i] = 0; });
        for (int i = 0; i < k; i++) {
            int next = rand_randn(*c.rng, main_area);
            while (flag[next]) next = rand_randn(*c.rng, main_area);
            obj_idxs[i] = next;
            flag[next] = 1;
        }
        int agent_x = obj_idxs[0] % h.main_width;
        int agent_y = obj_idxs[0] / h.main_width;
        a.x = (float)(agent_x + .5);
        a.y = (float)(agent_y + .5);
        {
            int16_t *g = c.grid;
            pg_warp_for(main_area, [=](int i) { g[i] = (int16_t)DIRT; });
        }
        for (int i = 0; i < num_diamonds; i++) E::set_obj_idx(c, obj_idxs[i + 1], DIAMOND);
        for (int i = 0; i < num_boulders; i++) E::set_obj_idx(c, obj_idxs[i + 1 + num_diamonds], BOULDER);
        int ndirt = 0;
        for (int i = 0; i < h.grid_size; i++)
            if (c.grid[i] == DIRT)
                dirt_cells[ndirt++] = i;
        E::set_obj(c, int(a.x), int(a.y), SPACE);
        for (int i = -1; i <= 1; i++)
            for (int j = -1; j <= 1; j++) {
                int ox = agent_x + i, oy = agent_y + j;
                if (E::get_obj(c, ox, oy) == BOULDER)
                    E::set_obj(c, ox, oy, DIRT);
            }
        int ncand = 0;
        for (int q = 0; q < ndirt; q++) {
            int cell = dirt_cells[q];
            int above_obj = E::get_obj_idx(c, cell + h.main_width);
            if (above_obj == DIRT || above_obj == c.oob)
                cands[ncand++] = cell;
        }
        if (ncand == 0) {
            h.err |= ERR_FASSERT;
            return;
        }
        int exit_cell = cands[rand_randn(*c.rng, ncand)];
        E::set_obj_idx(c, exit_cell, SPACE);
        int ei = E::add_entity(c, (float)((exit_cell % h.main_width) + .5), (float)((exit_cell / h.main_width) + .5), 0, 0, .5, EXIT);
        c.ents[ei].render_z = -1;
    }

    static PG_HD int get_moving_type(int type) { return type == DIAMOND ? MOVING_DIAMOND : (type == BOULDER ? MOVING_BOULDER : type); }
    static PG_HD bool is_moving(int type) { return type == MOVING_BOULDER || type == MOVING_DIAMOND; }
    static PG_HD int get_stationary_type(int type) { return type == MOVING_DIAMOND ? DIAMOND : (type == MOVING_BOULDER ? BOULDER : type); }
    static PG_HD bool is_round(int type) { return type == BOULDER || type == MOVING_BOULDER || type == DIAMOND || type == MOVING_DIAMOND; }
    static PG_HD bool is_free(Ctx &c, int idx) { return E::get_obj_idx(c, idx) == SPACE && (E::get_agent_index(c) != idx); }

    // miner.cpp:236-249
    static PG_HD void handle_push(Ctx &c) {
        EnvHdr &h = *c.h;
        Entity &a = agent_of(c);
        int agent_idx = E::get_agent_index(c);
        int agentx = agent_idx % h.main_width;
        if (h.action_vx == 1 && (a.vx == 0) && (agentx < h.main_width - 2) && E::get_obj_idx(c, agent_idx + 1) == BOULDER && E::get_obj_idx(c, agent_idx + 2) == SPACE) {
            E::set_obj_idx(c, agent_idx + 1, SPACE);
            E::set_obj_idx(c, agent_idx + 2, BOULDER);
            a.x += 1;
        } else if (h.action_vx == -1 && (a.vx == 0) && (agentx > 1) && E::get_obj_idx(c, agent_idx - 1) == BOULDER && E::get_obj_idx(c, agent_idx - 2) == SPACE) {
            E::set_obj_idx(c, agent_idx - 1, SPACE);
            E::set_obj_idx(c, agent_idx - 2, BOULDER);
            a.x -= 1;
        }
    }

    // miner.cpp:251-314. The full-grid gravity sweep only does work at round objects, so those are
    // located warp-wide; they are handled in ascending index order exactly like the serial loop
    // (an object rolled to idx+1 is revisited, as in the reference).
    static PG_HD void game_step(Ctx &c) {
        E::basic_game_step(c);
        EnvHdr &h = *c.h;
        Entity &a = agent_of(c);
        if (h.action_vx > 0)
            a.is_reflected = 0;
        if (h.action_vx < 0)
            a.is_reflected = 1;
        handle_push(c);
        int agent_obj = E::get_obj(c, int(a.x), int(a.y));
        if (agent_obj == DIAMOND)
            h.reward += DIAMOND_REWARD;
        if (agent_obj == DIRT || agent_obj == DIAMOND)
            E::set_obj(c, int(a.x), int(a.y), SPACE);
        const int main_area = h.main_width * h.main_height;
        const int W = h.main_width;
        int diamonds_count = 0;
        const int agent_idx = (int)(((double)a.y - .5) * W + ((double)a.x - .5));
        ScanUpIter it(0, main_area);
        while (true) {
            const int16_t *g = c.grid;
            const int idx = it.next([=](int i) {
                int o = g[i];
                return o == BOULDER || o == MOVING_BOULDER || o == DIAMOND || o == MOVING_DIAMOND;
            });
            if (idx < 0)
                break;
            int obj = E::get_obj_idx(c, idx);
            int obj_x = idx % W;
            int stat_type = get_stationary_type(obj);
            if (stat_type == DIAMOND)
                diamonds_count++;
            int below_idx = idx - W;
            int obj2 = E::get_obj_idx(c, below_idx);
            bool agent_is_below = agent_idx == below_idx;
            if (obj2 == SPACE && !agent_is_below) {
                E::set_obj_idx(c, idx, SPACE);
                E::set_obj_idx(c, below_idx, get_moving_type(obj));
            } else if (agent_is_below && is_moving(obj)) {
                h.done = 1;
            } else if (is_round(obj2) && obj_x > 0 && is_free(c, idx - 1) && is_free(c, idx - W - 1)) {
                E::set_obj_idx(c, idx, SPACE);
                E::set_obj_idx(c, idx - 1, get_stationary_type(obj));
            } else if (is_round(obj2) && obj_x < W - 1 && is_free(c, idx + 1) && is_free(c, idx - W + 1)) {
                E::set_obj_idx(c, idx, SPACE);
                E::set_obj_idx(c, idx + 1, stat_type);
                it.restart_from(idx + 1);  // the serial sweep meets the moved object again
            } else {
                E::set_obj_idx(c, idx, stat_type);
            }
        }
        st(c).diamonds_remaining = diamonds_count;
        for (int i = 0; i < h.n_ents; i++) {
            if (c.ents[i].type == ENEMY) {
                if (rand_randn(*c.rng, 6) == 0)
                    choose_new_vel(c, c.ents[i]);
            }
        }
    }
};

}  // namespace pg
