// Device game engine: episode lifecycle + 2-D physics/collision core shared by all games.
//
// Restates, for index-addressed POD state in HBM, what the reference does with a virtual class
// hierarchy over std::vector<std::shared_ptr<Entity>>:
//   Game::step/reset                      game.cpp:93-155
//   BasicAbstractGame::game_step & co.    basic-abstract-game.cpp:125-797, 1068-1150
//   Entity ctor/step                      entity.cpp:8-82
// Per-game behaviour is injected statically: `G` is a policy struct deriving from Defaults<G>
// (CRTP); a game "overrides" a hook by declaring a static function of the same name.  There is no
// virtual dispatch, no heap, no recursion deeper than the reference's own bound (push depth <= 5).
//
// Expression types (float vs double, int promotion) are kept exactly as in the reference line
// each function cites, because results must be bit-identical; see pg_common.cuh.
#pragma once
#include <type_traits>

#include "pg_bank.cuh"

namespace pg {

// ---------------------------------------------------------------- entity construction
// entity.cpp:11-51
PG_HD void entity_init(Entity &e, float x, float y, float vx, float vy, float rx, float ry, int type) {
    e.x = x;
    e.y = y;
    e.vx = vx;
    e.vy = vy;
    e.rx = rx;
    e.ry = ry;
    e.type = type;
    e.image_type = type;
    e.image_theme = 0;
    e.will_erase = 0;
    e.collides_with_entities = 0;
    e.collision_margin = 0.0f;
    e.rotation = 0.0f;
    e.is_reflected = 0;
    e.vrot = 0.0f;
    e.alpha = 1.0f;
    e.grow_rate = 1.0f;
    e.alpha_decay = 1.0f;
    e.fire_time = -1;
    e.spawn_time = -1;
    e.expire_time = -1;
    e.life_time = 0;
    e.health = 1;
    e.theta = -100;
    e.friction = 1;
    e.smart_step = 0;
    e.avoids_collisions = 0;
    e.auto_erase = 1;
    e.render_z = 0;
    e.use_abs_coords = 0;
    e.climber_spawn_x = 0;
    e.pad0 = 0;
    for (int i = 0; i < 5; i++) e.pad1[i] = 0;
    if (type == EXPLOSION) {
        e.grow_rate = 1.4f;
        e.expire_time = 4;
    } else if (type == TRAIL) {
        e.grow_rate = 1.05f;
        e.alpha_decay = 0.8f;
    }
}

// entity.cpp:57-82
PG_HD void entity_step(Entity &e) {
    if (!e.smart_step) {
        e.x += e.vx;
        e.y += e.vy;
    }
    e.rotation += e.vrot;
    e.vx *= e.friction;
    e.vy *= e.friction;
    e.life_time += 1;
    if (e.expire_time > 0 && e.life_time > e.expire_time) {
        e.will_erase = 1;
    }
    if (e.type == EXPLOSION) {
        if (e.image_type < EXPLOSION5) {
            e.image_type++;
        }
    }
    e.rx *= e.grow_rate;
    e.ry *= e.grow_rate;
    e.alpha = e.alpha_decay * e.alpha;
}

// entity.cpp:84-88. entity.cpp includes <math.h>, so this atan2 is the FLOAT function (atan2f in the
// oracle's object code) and the whole expression is float arithmetic; pg_atan2f reproduces the C
// library's (not correctly rounded) result bit for bit.
PG_HD void entity_face_direction(Entity &e, float dx, float dy, float rotation_offset = 0) {
    if (dx != 0 || dy != 0)
        e.rotation = -1 * pg_atan2f(dy, dx) + rotation_offset;
}

PG_HD Entity &agent_of(Ctx &c) { return c.ents[c.h->agent_idx]; }

// ---------------------------------------------------------------- Engine<G>
template <class G>
struct Engine {
    // ---- grid access (basic-abstract-game.cpp:167-218, grid.h)
    static PG_HD bool grid_contains(Ctx &c, int x, int y) {
        return 0 <= y && y < c.mh && 0 <= x && x < c.mw;
    }
    static PG_HD int get_obj(Ctx &c, int x, int y) {
        if (!grid_contains(c, x, y))
            return c.oob;
        return c.grid[y * c.mw + x];
    }
    static PG_HD int get_obj_idx(Ctx &c, int idx) {
        if (!(0 <= idx && idx < c.mw * c.mh))
            return c.oob;
        return c.grid[idx];
    }
    static PG_HD void set_obj(Ctx &c, int x, int y, int v) {
        if (!grid_contains(c, x, y)) {  // reference: fassert -> exit
            c.h->err |= ERR_GRID_OOB;
            return;
        }
        c.grid[y * c.mw + x] = (int16_t)v;
    }
    static PG_HD void set_obj_idx(Ctx &c, int idx, int v) {
        if (!(0 <= idx && idx < c.mw * c.mh)) {
            c.h->err |= ERR_GRID_OOB;
            return;
        }
        c.grid[idx] = (int16_t)v;
    }
    static PG_HD int to_grid_idx(Ctx &c, int x, int y) {
        if (!grid_contains(c, x, y))
            return INVALID_IDX;
        return y * c.mw + x;
    }
    // basic-abstract-game.cpp:125-131 (elem travels through a `char`). The cells are independent, so
    // the warp's lanes split the rectangle (level generation is the long tail of a step).
    static PG_HD void fill_elem(Ctx &c, int x, int y, int dx, int dy, int elem) {
        const int v = (int)(signed char)elem;
        if (dx <= 0 || dy <= 0)
            return;
        Ctx *cp = &c;
        pg_warp_for(dx * dy, [=](int k) {
            const int j = k / dy;
            set_obj(*cp, x + j, y + (k - j * dy), v);
        });
    }
    // basic-abstract-game.cpp:167-174 — floor() is the double overload
    static PG_HD int get_obj_from_floats(Ctx &c, float i, float j) {
        if (i < 0)
            return c.oob;
        if (j < 0)
            return c.oob;
        return get_obj(c, (int)pg_dfloor((double)i), (int)pg_dfloor((double)j));
    }
    static PG_HD int get_agent_index(Ctx &c) {
        Entity &a = agent_of(c);
        return int(a.y) * c.mw + int(a.x);
    }

    // ---- entity list
    static PG_HD int push_entity(Ctx &c) {
        int n = c.h->n_ents;
        if (n >= c.ent_cap) {
            c.h->err |= ERR_ENTITY_OVERFLOW;
            return c.ent_cap - 1;  // overwrite the last slot; error is latched and reported
        }
        c.h->n_ents = n + 1;
        if (n + 1 > c.h->max_ents_seen)
            c.h->max_ents_seen = n + 1;
        return n;
    }
    // basic-abstract-game.cpp:563-573
    static PG_HD int add_entity_rxy(Ctx &c, float x, float y, float vx, float vy, float rx, float ry, int type) {
        int i = push_entity(c);
        entity_init(c.ents[i], x, y, vx, vy, rx, ry, type);
        return i;
    }
    static PG_HD int add_entity(Ctx &c, float x, float y, float vx, float vy, float r, int type) {
        return add_entity_rxy(c, x, y, vx, vy, r, r, type);
    }
    // basic-abstract-game.cpp:575-582
    static PG_HD int spawn_entity_at_idx(Ctx &c, int idx, float r, int type) {
        float x = (idx % c.mw) + .5;
        float y = (idx / c.mw) + .5;
        return add_entity(c, x, y, 0, 0, r, type);
    }
    // basic-abstract-game.cpp:225-231
    static PG_HD int spawn_child(Ctx &c, int src, int type, float obj_r, bool match_vel = false) {
        float vx = match_vel ? c.ents[src].vx : 0;
        float vy = match_vel ? c.ents[src].vy : 0;
        float sx = c.ents[src].x, sy = c.ents[src].y;
        return add_entity(c, sx, sy, vx, vy, obj_r, type);
    }

    // ---- collision predicates
    // basic-abstract-game.cpp:1145-1150 — fabs is the double overload; thresholds are float sums
    static PG_HD bool has_collision(const Entity &e1, const Entity &e2, float margin) {
        float threshold_x = (e1.rx + e2.rx) + margin;
        float threshold_y = (e1.ry + e2.ry) + margin;
        return (pg_dfabs((double)(e1.x - e2.x)) < (double)threshold_x) && (pg_dfabs((double)(e1.y - e2.y)) < (double)threshold_y);
    }
    // basic-abstract-game.cpp:1126-1131
    static PG_HD bool has_agent_collision(Ctx &c, const Entity &e1) {
        if (e1.type == PLAYER)
            return false;
        return has_collision(e1, agent_of(c), e1.collision_margin);
    }
    // basic-abstract-game.cpp:1114-1124
    static PG_HD bool has_any_collision(Ctx &c, const Entity &e1, float margin = 0) {
        const Entity *ents = c.ents;
        return pg_scan_down(c.h->n_ents, [&](int i) {
                   const Entity &ent = ents[i];
                   return !ent.avoids_collisions && has_collision(e1, ent, margin);
               }) >= 0;
    }
    // basic-abstract-game.cpp:520-528
    static PG_HD bool agent_has_collision(Ctx &c) {
        Ctx *cp = &c;
        return pg_scan_down(c.h->n_ents, [&](int i) { return has_agent_collision(*cp, cp->ents[i]); }) >= 0;
    }
    // basic-abstract-game.cpp:1068-1084
    static PG_HD bool is_out_of_bounds(Ctx &c, const Entity &e1) {
        float x = e1.x, y = e1.y, rx = e1.rx, ry = e1.ry;
        if (x + rx < 0)
            return true;
        if (y + ry < 0)
            return true;
        if (x - rx > c.mw)
            return true;
        if (y - ry > c.mh)
            return true;
        return false;
    }
    // basic-abstract-game.cpp:133-143
    static PG_HD float get_distance(const Entity &p0, const Entity &p1) {
        float dx = p0.x - p1.x;
        float dy = p0.y - p1.y;
        return (float)pg_dsqrt((double)(dx * dx + dy * dy));
    }
    // basic-abstract-game.cpp:1133-1143
    static PG_HD int find_entity_index(Ctx &c, int type) {
        int index = -1;
        for (int i = 0; i < c.h->n_ents; i++)
            if (c.ents[i].type == type)
                index = i;
        return index;
    }

    // ---- random placement (basic-abstract-game.cpp:511-561, 1100-1112)
    static PG_HD float rand_pos(Ctx &c, float r, float min, float max) {
        if (max - min <= 2 * r)
            return (max + min) / 2;
        float range = max - min;
        return (range - 2 * r) * rand_rand01(*c.rng) + r + min;
    }
    static PG_HD void reposition(Ctx &c, int ei, float x, float y, float w, float h, bool check_collisions) {
        Entity &ent = c.ents[ei];
        float rx = ent.rx, ry = ent.ry;
        ent.x = rand_pos(c, rx, x, x + w);
        ent.y = rand_pos(c, ry, y, y + h);
        int count = 0;
        while ((has_agent_collision(c, ent) || (check_collisions && has_any_collision(c, ent))) && (count < 100)) {
            ent.x = rand_pos(c, rx, x, x + w);
            ent.y = rand_pos(c, ry, y, y + h);
            count++;
        }
    }
    // basic-abstract-game.cpp:511-518: the entity is built, placed against the CURRENT list, then
    // appended (so it never tests against itself)
    static PG_HD int spawn_entity_rxy(Ctx &c, float rx, float ry, int type, float x, float y, float w, float h, bool check_collisions = true) {
        int n = c.h->n_ents;
        if (n >= c.ent_cap) {
            c.h->err |= ERR_ENTITY_OVERFLOW;
            return c.ent_cap - 1;
        }
        entity_init(c.ents[n], 0, 0, 0, 0, rx, ry, type);
        reposition(c, n, x, y, w, h, check_collisions);  // list length still n: slot n is not scanned
        return push_entity(c);
    }
    static PG_HD int spawn_entity(Ctx &c, float r, int type, float x, float y, float w, float h, bool check_collisions = true) {
        return spawn_entity_rxy(c, r, r, type, x, y, w, h, check_collisions);
    }
    static PG_HD void spawn_entities(Ctx &c, int num, float r, int type, float x, float y, float w, float h) {
        for (int i = 0; i < num; i++)
            spawn_entity(c, r, type, x, y, w, h);
    }
    static PG_HD void reposition_agent(Ctx &c) {
        int count = 0;
        Entity &a = agent_of(c);
        do {
            a.x = rand_rand01(*c.rng) * (c.h->main_width - 2 * a.rx) + a.rx;
            a.y = rand_rand01(*c.rng) * (c.h->main_height - 2 * a.ry) + a.ry;
            count++;
        } while (agent_has_collision(c) && (count < 100));
    }

    // ---- themes / aspect ratios (basic-abstract-game.cpp:1014-1046)
    static PG_HD void choose_random_theme(Ctx &c, Entity &ent) {
        ent.image_theme = rand_randn(*c.rng, c.assets->num_themes[ent.image_type]);
    }
    static PG_HD void choose_step_random_theme(Ctx &c, Entity &ent) {
        ent.image_theme = c.h->step_rand_int % c.assets->num_themes[ent.image_type];
    }
    // initialize_asset_if_necessary (basic-abstract-game.cpp:79-123) fills slot [type + 100 * theme] with
    // the image of the MASKED theme (:86), so under restrict_themes the aspect ratio game logic reads
    // for any theme is theme 0's
    static PG_HD int asset_slot(Ctx &c, const Entity &ent) {
        int theme = ent.image_theme;
        if (c.h->options.restrict_themes && !G::should_preserve_type_themes(c, ent.image_type))
            theme = 0;
        return ent.image_type + theme * MAX_ASSETS;
    }
    static PG_HD void match_aspect_ratio(Ctx &c, Entity &ent, bool match_width = true) {
        int img_idx = asset_slot(c, ent);
        if (match_width)
            ent.ry = ent.rx / c.assets->aspect[img_idx];
        else
            ent.rx = ent.ry * c.assets->aspect[img_idx];
    }
    static PG_HD void fit_aspect_ratio(Ctx &c, Entity &ent) {
        int img_idx = asset_slot(c, ent);
        float ar = c.assets->aspect[img_idx];
        if (ar > 1)
            ent.ry = ent.rx / ar;
        else
            ent.rx = ent.ry * ar;
    }

    // ---- physics
    // basic-abstract-game.cpp:240-268. sign() is double, so the offset is evaluated in double.
    // push_obj and sub_step call each other (bounded recursion), so they are real functions and the env
    // handle they get by reference lives in the caller's local memory: every c.grid / c.mw / c.ents
    // read through it is a stack load (measured: two thirds of the logic kernel's L1 requests). Each
    // works on a private copy instead — only the fields it uses are loaded, once per call. (Passing
    // the handle by value was measured too: the 27-word copy at every call site costs more.)
    static PG_HD_NOINLINE bool push_obj(Ctx &cref, int src, int target, bool is_horizontal, int depth) {
        Ctx c = cref;
        Entity &s = c.ents[src];
        Entity &t = c.ents[target];
        float rsum = is_horizontal ? (s.rx + t.rx) : (s.ry + t.ry);
        float delx = t.x - s.x;
        float dely = t.y - s.y;
        float t_vx = 0;
        float t_vy = 0;
        if (is_horizontal)
            t_vx = (float)((double)s.x + pg_sign((double)delx) * (double)rsum - (double)t.x);
        else
            t_vy = (float)((double)s.y + pg_sign((double)dely) * (double)rsum - (double)t.y);
        bool block = false;
        if (depth < 5)
            block = sub_step(cref, target, t_vx, t_vy, depth + 1);
        if (is_horizontal)
            t.vx = 0;
        else
            t.vy = 0;
        return block;
    }

    // basic-abstract-game.cpp:270-372
    // out-of-line entry for the recursion push_obj -> sub_step (crates pushing crates); the first level
    // is inlined into basic_step_object: called 8+ times per smart entity and step, a real call there
    // spent a third of the kernel's stack traffic on saving and restoring registers
    static PG_HD_NOINLINE bool sub_step(Ctx &cref, int oi, float _vx, float _vy, int depth) {
        Ctx c = cref;
        return sub_step_impl(c, oi, _vx, _vy, depth);
    }
    static PG_HD bool sub_step_impl(Ctx &c, int oi, float _vx, float _vy, int depth) {
        Entity &obj = c.ents[oi];
        if (obj.will_erase)
            return false;

        float ny = obj.y + _vy;
        float nx = obj.x + _vx;
        float margin = 0.98f;
        bool is_horizontal = _vx != 0;
        bool block = false;
        bool reflect = false;

        for (int i = 0; i < 2; i++) {
            for (int j = 0; j < 2; j++) {
                int type2 = get_obj_from_floats(c, nx + obj.rx * margin * (2 * i - 1), ny + obj.ry * margin * (2 * j - 1));
                block = block || G::is_blocked(c, oi, type2, is_horizontal);
                reflect = reflect || G::will_reflect(c, obj.type, type2);
            }
        }

        const bool grid_step = c.h->grid_step != 0;

        if (reflect) {
            if (is_horizontal) {
                float delta;
                if (_vx < 0)
                    delta = (float)(pg_dceil((double)(nx - obj.rx)) - (double)(nx - obj.rx));
                else
                    delta = (float)(pg_dfloor((double)(nx + obj.rx)) - (double)(nx + obj.rx));
                obj.vx = -1 * obj.vx;
                nx = nx + 2 * delta;
            } else {
                float delta;
                if (_vy < 0)
                    delta = (float)(pg_dceil((double)(ny - obj.ry)) - (double)(ny - obj.ry));
                else
                    delta = (float)(pg_dfloor((double)(ny + obj.ry)) - (double)(ny + obj.ry));
                obj.vy = -1 * obj.vy;
                ny = ny + 2 * delta;
            }
        } else if (block) {
            if (is_horizontal) {
                if (grid_step)
                    nx = obj.x;
                else
                    nx = (float)(_vx > 0 ? (pg_dfloor((double)(nx + obj.rx)) - (double)obj.rx) : (pg_dceil((double)(nx - obj.rx)) + (double)obj.rx));
            } else {
                if (grid_step)
                    ny = obj.y;
                else
                    ny = (float)(_vy > 0 ? (pg_dfloor((double)(ny + obj.ry)) - (double)obj.ry) : (pg_dceil((double)(ny - obj.ry)) + (double)obj.ry));
            }
        }

        obj.x = nx;
        obj.y = ny;

        bool block2 = false;

        // reference: for i = n-1..0 { skip self/erased; if (has_collision) {...} } — the test runs
        // warp-wide, the (rare) hits are handled one at a time in descending order, and the scan
        // restarts below each hit because handling may have moved things.
        ScanDownIter it((c.obst_hi >= 0 && c.obst_hi < c.h->n_ents) ? c.obst_hi : c.h->n_ents);
        while (true) {
            const Entity *ents = c.ents;
            const float ox = obj.x, oy = obj.y, orx = obj.rx, ory = obj.ry;  // hoisted: warp-uniform
            const int otype = obj.type;
            Ctx &cp0 = c;
            const int i = it.next([&](int k) {
                const Entity &mm = ents[k];
                if (k == oi || mm.will_erase)
                    return false;
                // overlaps that can neither block nor reflect change nothing (:332-356); games may
                // declare such type pairs so they are dropped inside the warp-wide test
                if (!G::may_block_or_reflect(cp0, otype, mm.type))
                    return false;
                // has_collision(obj, m, POS_EPS), basic-abstract-game.cpp:1145-1150
                float threshold_x = (orx + mm.rx) + POS_EPS;
                float threshold_y = (ory + mm.ry) + POS_EPS;
                return (pg_dfabs((double)(ox - mm.x)) < (double)threshold_x) && (pg_dfabs((double)(oy - mm.y)) < (double)threshold_y);
            });
            if (i < 0)
                break;
            Entity &m = c.ents[i];
            bool curr_block = false;
            bool moved = false;
            if (G::is_blocked_ents(c, oi, i, is_horizontal)) {
                curr_block = true;
            } else if (G::will_reflect(c, obj.type, m.type)) {
                moved = true;
                if (is_horizontal) {
                    float delx = m.x - obj.x;
                    float rsum = m.rx + obj.rx;
                    obj.x += _vx > 0 ? -2 * (rsum - delx) : 2 * (rsum + delx);
                    obj.vx = -1 * obj.vx;
                } else {
                    float dely = m.y - obj.y;
                    float rsum = m.ry + obj.ry;
                    obj.y += _vy > 0 ? -2 * (rsum - dely) : 2 * (rsum + dely);
                    obj.vy = -1 * obj.vy;
                }
            }
            if (curr_block) {
                Ctx cp = c;  // only this copy's address leaves the function
                push_obj(cp, i, oi, is_horizontal, depth);
                moved = true;
            }
            block2 = block2 || curr_block;
            // positions / erase flags may have changed: the remaining ballot bits are stale
            if (moved)
                it.restart_below(i);
        }
        return block || block2;
    }

    // basic-abstract-game.cpp:593-656
    static PG_HD void basic_step_object(Ctx &c, int oi) {
        Entity &obj = c.ents[oi];
        if (obj.will_erase)
            return;
        int num_sub_steps;
        if (c.h->grid_step) {
            num_sub_steps = 1;
        } else {
            num_sub_steps = int(4 * pg_dsqrt((double)(obj.vx * obj.vx + obj.vy * obj.vy)));
            if (num_sub_steps < 4)
                num_sub_steps = 4;
        }
        float pct = (float)(1.0 / num_sub_steps);
        float cmp = (float)(pg_dfabs((double)obj.vx) - pg_dfabs((double)obj.vy));
        bool step_x_first = cmp == 0 ? c.h->step_rand_int % 2 == 0 : (cmp > 0);
        if (obj.type == PLAYER) {
            if (c.h->action_vx != 0)
                step_x_first = true;
            if (c.h->action_vy != 0)
                step_x_first = false;
        }
        float vx_pct = 0;
        float vy_pct = 0;
        for (int s = 0; s < num_sub_steps; s++) {
            bool block_x = false;
            bool block_y = false;
            // x then y, or y then x: one inlined copy of the sub-step body, run twice
            for (int half = 0; half < 2; half++) {
                const bool do_x = (half == 0) == step_x_first;
                const bool blocked = sub_step_impl(c, oi, do_x ? obj.vx * pct : 0.0f, do_x ? 0.0f : obj.vy * pct, 0);
                if (do_x)
                    block_x = blocked;
                else
                    block_y = blocked;
            }
            if (!block_x)
                vx_pct += 1;
            if (!block_y)
                vy_pct += 1;
            if (block_x && block_y)
                break;
        }
        vx_pct = vx_pct / num_sub_steps;
        vy_pct = vy_pct / num_sub_steps;
        obj.vx *= vx_pct;
        obj.vy *= vy_pct;
    }

    // basic-abstract-game.cpp:1086-1098 (`given` is always the live list; the count is latched).
    // The reference walks the list from the back: smart_step entities run the sub-step physics
    // (which reads every other entity), all others just integrate their own fields. Entities that
    // only integrate commute with each other, so each run of them between two smart entities is
    // stepped by the warp's lanes in parallel; smart entities keep their place in the order.
    static PG_HD void step_entities(Ctx &c) {
        int hi = c.h->n_ents;
        {
            // no entity is added, erased, moved in the list or re-typed while entities are stepped
            Ctx *cp = &c;
            const Entity *ents0 = c.ents;
            c.obst_hi = 1 + pg_scan_down(hi, [=](int k) { return G::may_be_obstacle(*cp, ents0[k].type); });
        }
        while (hi > 0) {
            Entity *ents = c.ents;
            const int s = pg_scan_down(hi, [=](int k) { return ents[k].smart_step != 0; });
            const int lo = s + 1;  // entities [lo, hi) only integrate
            pg_warp_for(hi - lo, [=](int k) { entity_step(ents[lo + k]); });
            if (s < 0)
                break;
            basic_step_object(c, s);
            entity_step(c.ents[s]);
            hi = s;
        }
        c.obst_hi = -1;
    }

    // basic-abstract-game.cpp:145-165
    static PG_HD void check_grid_collisions(Ctx &c, int ei) {
        Entity &ent = c.ents[ei];
        float ax = ent.x, ay = ent.y, arx = ent.rx, ary = ent.ry;
        int min_x = int(ax - (arx + POS_EPS));
        int max_x = int(ax + (arx + POS_EPS));
        int min_y = int(ay - (ary + POS_EPS));
        int max_y = int(ay + (ary + POS_EPS));
        for (int x = min_x; x <= max_x; x++) {
            for (int y = min_y; y <= max_y; y++) {
                int grid_type = get_obj_from_floats(c, (float)x, (float)y);
                if (grid_type != SPACE)
                    G::handle_grid_collision(c, ei, grid_type, x, y);
            }
        }
    }

    // basic-abstract-game.cpp:748-756. Order-preserving compaction; an erased agent moves to the
    // ghost slot so later reads through `agent` still work (the reference keeps it alive via
    // shared_ptr). On the device each lane owns one entity of a 32-entity chunk: the erase tests
    // run in parallel, a ballot + popcount gives every survivor its destination, all lanes read
    // their record before any lane writes (destinations never lie beyond the chunk's sources),
    // and the per-game bookkeeping hooks then run in list order, warp-uniformly.
    static PG_HD void erase_if_needed(Ctx &c) {
        const int n = c.h->n_ents;
        int w = 0;
        int agent_idx = c.h->agent_idx;
#if defined(__CUDA_ARCH__)
        const int lane = (int)(threadIdx.x & 31u);
        const int old_agent = c.h->agent_idx;
        // common case first: nothing to erase
        {
            Ctx *cp = &c;
            ScanUpIter it(0, n);
            const int first = it.next([=](int k) {
                const Entity &e = cp->ents[k];
                return e.will_erase || (e.auto_erase && is_out_of_bounds(*cp, e));
            });
            if (first < 0)
                return;
            w = first & ~31;  // whole chunks before the first erased entity stay where they are
        }
        for (int base = w; base < n; base += 32) {
            const int i = base + lane;
            const bool valid = i < n;
            Entity e;
            bool erase = false;
            if (valid) {
                e = c.ents[i];
                erase = e.will_erase || (e.auto_erase && is_out_of_bounds(c, e));
            }
            const unsigned keepmask = __ballot_sync(0xffffffffu, valid && !erase);
            const unsigned erasemask = __ballot_sync(0xffffffffu, erase);
            const int dest = w + __popc(keepmask & ((1u << lane) - 1u));
            __syncwarp();
            if (valid && !erase && dest != i)
                c.ents[dest] = e;
            if (valid && i == old_agent && erase)
                c.ents[c.ent_cap] = e;
            const unsigned agent_lane_mask = __ballot_sync(0xffffffffu, valid && i == old_agent);
            if (agent_lane_mask) {
                const int al = __ffs((int)agent_lane_mask) - 1;
                const int adest = __shfl_sync(0xffffffffu, dest, al);
                agent_idx = ((erasemask >> al) & 1u) ? c.ent_cap : adest;
            }
            __syncwarp();
            if (G::HAS_ENTITY_HOOKS) {
                unsigned touched = erasemask | keepmask;
                while (touched) {
                    const int l = __ffs((int)touched) - 1;
                    touched &= touched - 1;
                    const int src = base + l;
                    if ((erasemask >> l) & 1u) {
                        G::on_entity_erased(c, src);
                    } else {
                        const int d = __shfl_sync(0xffffffffu, dest, l);
                        if (d != src)
                            G::on_entity_moved(c, src, d);
                    }
                }
            }
            w += __popc(keepmask);
        }
#else
        for (int i = 0; i < n; i++) {
            Entity &e = c.ents[i];
            bool erase = e.will_erase || (e.auto_erase && is_out_of_bounds(c, e));
            if (erase) {
                if (i == c.h->agent_idx) {
                    c.ents[c.ent_cap] = e;
                    agent_idx = c.ent_cap;
                }
                G::on_entity_erased(c, i);
                continue;
            }
            if (w != i) {
                c.ents[w] = e;
                if (i == c.h->agent_idx)
                    agent_idx = w;
                G::on_entity_moved(c, i, w);
            }
            w++;
        }
#endif
        c.h->n_ents = w;
        c.h->agent_idx = agent_idx;
    }

    // basic-abstract-game.cpp:664-684
    static PG_HD void decay_agent_velocity(Ctx &c) {
        Entity &a = agent_of(c);
        a.vx = (float)(.9 * a.vx);
        a.vy = (float)(.9 * a.vy);
    }
    static PG_HD void default_update_agent_velocity(Ctx &c) {
        EnvHdr &h = *c.h;
        Entity &a = agent_of(c);
        float v_scale = G::get_agent_acceleration_scale(c);
        a.vx = (1 - h.mixrate) * a.vx;
        a.vy = (1 - h.mixrate) * a.vy;
        a.vx += h.mixrate * h.maxspeed * h.action_vx * v_scale;
        a.vy += h.mixrate * h.maxspeed * h.action_vy * v_scale;
        decay_agent_velocity(c);
    }

    // basic-abstract-game.cpp:686-746
    static PG_HD void basic_game_step(Ctx &c) {
        EnvHdr &h = *c.h;
        PG_PHASE_RESET(c);
        PG_PHASE_BEGIN(c);
        h.step_rand_int = rand_randint(*c.rng, 0, 1000000);
        h.move_action = h.action % 9;
        h.special_action = 0;
        if (h.action >= 9) {
            h.special_action = h.action - 8;
            h.move_action = 4;
        }
        if (h.move_action != 4)
            h.last_move_action = h.move_action;
        h.action_vrot = 0;
        h.action_vx = 0;
        h.action_vy = 0;
        G::set_action_xy(c, h.move_action);

        if (h.grid_step) {
            Entity &a = agent_of(c);
            a.vx = h.action_vx;
            a.vy = h.action_vy;
        } else {
            G::update_agent_velocity(c);
            Entity &a = agent_of(c);
            a.vrot = MIXRATEROT * a.vrot;
            a.vrot += MIXRATEROT * MAXVTHETA * h.action_vrot;
        }

        PG_PHASE_END(c, 0);
        step_entities(c);
        PG_PHASE_END(c, 1);

        // collision pass (:719-741): entities that need any work are found warp-wide; each is then
        // processed exactly as the reference's loop body, in descending order.
        int i = h.n_ents;
        while (true) {
            Ctx *cp = &c;
            i = pg_scan_down(i, [&](int k) {
                const Entity &e = cp->ents[k];
                return e.collides_with_entities || e.smart_step || has_agent_collision(*cp, e);
            });
            if (i < 0)
                break;
            if (has_agent_collision(c, c.ents[i]))
                G::handle_agent_collision(c, i);
            if (c.ents[i].collides_with_entities) {
                int j = h.n_ents;
                while (true) {
                    j = pg_scan_down(j, [&](int k) {
                        const Entity &a = cp->ents[i];
                        const Entity &b = cp->ents[k];
                        return k != i && has_collision(a, b, a.collision_margin) && !a.will_erase && !b.will_erase;
                    });
                    if (j < 0)
                        break;
                    G::handle_collision(c, i, j);
                }
            }
            if (c.ents[i].smart_step)
                check_grid_collisions(c, i);
        }

        PG_PHASE_END(c, 2);
        erase_if_needed(c);
        h.done = h.done || is_out_of_bounds(c, agent_of(c));
        PG_PHASE_END(c, 3);
        PG_PHASE_NOTE(c, 4, h.n_ents);
    }

    // basic-abstract-game.cpp:758-797
    static PG_HD void basic_game_reset(Ctx &c) {
        EnvHdr &h = *c.h;
        G::choose_world_dim(c);
        ctx_refresh(c);
        h.bg_pct_x = rand_rand01(*c.rng);
        h.grid_size = h.main_width * h.main_height;
        if (h.grid_size > c.grid_cap) {
            h.err |= ERR_GRID_OOB;
            h.main_width = 1;
            h.main_height = 1;
            h.grid_size = 1;
            ctx_refresh(c);
        }
        h.background_index = rand_randn(*c.rng, c.assets->num_backgrounds);
        h.n_ents = 0;
        float ax, ay;
        float a_r = 0.4f;
        if (h.random_agent_start) {
            ax = rand_rand01(*c.rng) * (h.main_width - 2 * a_r) + a_r;
            ay = rand_rand01(*c.rng) * (h.main_height - 2 * a_r) + a_r;
        } else {
            ax = a_r;
            ay = a_r;
        }
        h.agent_idx = 0;
        int ai = add_entity(c, ax, ay, 0, 0, a_r, PLAYER);
        c.ents[ai].smart_step = 1;
        c.ents[ai].render_z = 1;
        erase_if_needed(c);
        // grid.resize() zero-fills, then fill_elem(..., SPACE)
        {
            int16_t *g = c.grid;
            pg_warp_for(h.grid_size, [=](int i) { g[i] = (int16_t)SPACE; });
        }
    }

    // ---- Game::reset / Game::step (game.cpp:93-155)
    // level_seed_override >= 0 (pgb200_get_next_level_seeds) replaces the draw of the next level seed and
    // nothing else: level_seed_rand_gen is not advanced. Returns whether the override was taken.
    // BANK: a level the bank holds (bank_copy_level) is copied instead of generated; nothing else changes.
    // Source (level lookahead): src->copy_level(c) decides instead whether the level is copied, and from where.
    template <bool BANK = false, class Source = void>
    static PG_HD bool reset(Ctx &c, int32_t level_seed_override = -1, const LevelBank *bank = nullptr, const Source *src = nullptr) {
        EnvHdr &h = *c.h;
        bool took = false;
        h.reset_count++;
        if (h.episodes_remaining == 0) {
            if (level_seed_override >= 0) {
                h.current_level_seed = level_seed_override;
                took = true;
            } else if (h.options.use_sequential_levels && h.level_complete) {
                h.current_level_seed = (int32_t)((uint32_t)h.current_level_seed + 997u);
            } else {
                h.current_level_seed = rand_randint(*c.lvl_rng, h.level_seed_low, h.level_seed_high);
            }
            h.episodes_remaining = 1;
        } else {
            h.reward = 0;
            h.done = 0;
            h.level_complete = 0;
        }
        bool generate;
        if constexpr (std::is_void<Source>::value)
            generate = !BANK || !bank_copy_level<G>(c, *bank);
        else
            generate = !src->copy_level(c);
        if (generate) {
            mt_seed(*c.rng, (uint32_t)h.current_level_seed);
            G::game_reset(c);
        }
        h.cur_time = 0;
        h.total_reward = 0;
        h.episodes_remaining -= 1;
        h.action = h.default_action;
        return took;
    }

    // Game::step (game.cpp:120-155) in two halves, so that the vector runtime can run level generation
    // (the reset of an episode that just ended) as a separate pass: step_play = everything up to the
    // decision `if (step_data.done) reset()`, returns that decision; step_finish = the rest, returns whether
    // its reset took level_seed_override.
    // level_end (pgb200_get_final_outputs): receives why the level ends in this step, in the order of the
    // `done` expression below: PGB200_LEVEL_END_GAME, _TIMEOUT, _CALLER, or 0 when it does not end.
    template <bool CAUSE = false>
    static PG_HD bool step_play(Ctx &c, uint8_t *level_end = nullptr) {
        EnvHdr &h = *c.h;
        h.cur_time += 1;
        bool will_force_reset = false;
        if (h.action == -1) {
            h.action = h.default_action;
            will_force_reset = true;
        }
        h.reward = 0;
        h.done = 0;
        h.level_complete = 0;
        G::game_step(c);
        if (CAUSE)
            *level_end = h.done ? 1 : (h.cur_time >= h.timeout ? 2 : (will_force_reset ? 3 : 0));
        h.done = h.done || will_force_reset || (h.cur_time >= h.timeout);
        h.total_reward += h.reward;
        if (h.reward != 0) {
            h.last_reward_timer = 10;
            h.last_reward = h.reward;
        }
        h.prev_level_seed = h.current_level_seed;
        return h.done != 0;
    }
    template <bool BANK = false, class Source = void>
    static PG_HD bool step_finish(Ctx &c, bool do_reset, int32_t level_seed_override, const LevelBank *bank = nullptr,
                                  const Source *src = nullptr) {
        EnvHdr &h = *c.h;
        bool took = false;
        if (do_reset)
            took = reset<BANK, Source>(c, level_seed_override, bank, src);
        if (h.options.use_sequential_levels && h.level_complete)
            h.done = 0;
        h.episode_done = h.done;
        return took;
    }
    static PG_HD void step(Ctx &c) { step_finish(c, step_play(c), -1); }
};

// ---------------------------------------------------------------- default hooks (the virtuals)
template <class G>
struct Defaults {
    using E = Engine<G>;
    // constructor-time constants (BasicAbstractGame ctor, basic-abstract-game.cpp:22-46; Game ctor
    // game.cpp:25-39). Games shadow `init_constants` and call this first.
    static PG_HD void base_init_constants(Ctx &c) {
        EnvHdr &h = *c.h;
        h.timeout = 1000;
        h.episodes_remaining = 0;
        h.last_reward = -1;
        h.last_reward_timer = 0;
        h.fixed_asset_seed = 0;
        h.reset_count = 0;
        h.current_level_seed = 0;
        h.prev_level_seed = 0;
        h.reward = 0;
        h.done = 1;
        h.level_complete = 0;
        h.episode_done = 0;
        h.cur_time = 0;
        h.total_reward = 0;
        h.action = 0;
        h.grid_step = 0;
        h.initial_reset_complete = 0;
        h.char_dim = 5;
        h.main_width = 0;
        h.main_height = 0;
        h.visibility = 16;
        h.min_visibility = 0;
        h.mixrate = 0.5;
        h.maxspeed = 0.5;
        h.max_jump = h.maxspeed;
        h.default_action = 4;
        h.last_move_action = 7;
        h.move_action = 0;
        h.special_action = 0;
        h.bg_tile_ratio = 0;
        h.bg_pct_x = 0;
        h.background_index = 0;
        h.out_of_bounds_object = INVALID_OBJ;
        h.has_useful_vel_info = 1;
        h.random_agent_start = 1;
        h.action_vx = h.action_vy = h.action_vrot = 0;
        h.center_x = h.center_y = 0;
        h.step_rand_int = 0;
        h.unit = h.view_dim = h.x_off = h.y_off = 0;
        h.grid_size = 0;
        h.n_ents = 0;
        h.agent_idx = 0;
        h.err = 0;
        h.max_ents_seen = 0;
        h.max_blits_seen = 0;
        h.max_rots_seen = 0;
        for (int i = 0; i < GAME_STATE_BYTES; i++) h.game_state[i] = 0;
    }
    static PG_HD void init_constants(Ctx &c) { base_init_constants(c); }

    // basic-abstract-game.cpp:482-497
    static PG_HD bool is_blocked(Ctx &c, int src, int target, bool is_horizontal) {
        if (target == WALL_OBJ)
            return true;
        if (target == c.oob)
            return true;
        return false;
    }
    static PG_HD bool is_blocked_ents(Ctx &c, int src, int target, bool is_horizontal) {
        return G::is_blocked(c, src, c.ents[target].type, is_horizontal);
    }
    static PG_HD bool will_reflect(Ctx &c, int src_type, int target_type) { return false; }
    // PURE, conservative pre-filter for sub_step's entity scan: false only if an overlap between
    // entities of these two types can never make is_blocked_ents or will_reflect return true.
    static PG_HD bool may_block_or_reflect(Ctx &c, int src_type, int target_type) { return true; }
    // PURE, conservative: false only if NO source type can be blocked or reflected by an entity of
    // this type (may_block_or_reflect(s, target_type) is false for every s). step_entities uses it
    // to bound sub_step's entity scans to the list prefix that contains such entities at all — in
    // coinrun only crates qualify, and they sit in front of the hundreds of trail entities that a
    // level with many enemies accumulates.
    static PG_HD bool may_be_obstacle(Ctx &c, int target_type) { return true; }
    static PG_HD float get_agent_acceleration_scale(Ctx &c) { return 1.0; }
    static PG_HD void handle_agent_collision(Ctx &c, int obj) {}
    static PG_HD void handle_grid_collision(Ctx &c, int obj, int type, int i, int j) {}
    static PG_HD void handle_collision(Ctx &c, int src, int target) {}
    static PG_HD void choose_world_dim(Ctx &c) {}
    // basic-abstract-game.cpp:658-662
    static PG_HD void set_action_xy(Ctx &c, int move_act) {
        c.h->action_vx = move_act / 3 - 1;
        c.h->action_vy = move_act % 3 - 1;
        c.h->action_vrot = 0;
    }
    static PG_HD void update_agent_velocity(Ctx &c) { E::default_update_agent_velocity(c); }
    static PG_HD void game_step(Ctx &c) { E::basic_game_step(c); }
    static PG_HD void game_reset(Ctx &c) { E::basic_game_reset(c); }
    // scratch words [PERSIST_SCRATCH_FIRST, + PERSIST_SCRATCH_WORDS) outlive game_reset (the game's steps or its
    // state blob read them); every other scratch word is level-generation workspace. A banked level carries these.
    static constexpr int PERSIST_SCRATCH_FIRST = 0;
    static constexpr int PERSIST_SCRATCH_WORDS = 0;
    // bytes [STEP_STATE_OFFSET, + STEP_STATE_BYTES) of the game's state struct (game_state) are written by its steps
    // and never by game_reset, so that a reset inherits them from the episode before; a banked level leaves them be
    static constexpr int STEP_STATE_OFFSET = 0;
    static constexpr int STEP_STATE_BYTES = 0;
    // bookkeeping hooks for games that hold references to entities (shared_ptr members); a game
    // that defines them sets HAS_ENTITY_HOOKS
    static constexpr bool HAS_ENTITY_HOOKS = false;
    static PG_HD void on_entity_moved(Ctx &c, int from, int to) {}
    static PG_HD void on_entity_erased(Ctx &c, int idx) {}

    // ---- draw-side hooks (basic-abstract-game.cpp:432-446, 799-817, 1048-1050)
    // false = the game never writes its grid (all SPACE) and always draws the whole world
    // (center_agent forced off): the frame then carries no cell blits at all
    static constexpr bool DRAWS_GRID = true;
    // > 0: the game honours center_agent = false by drawing its whole world (basic-abstract-game.cpp:
    // 819-838); cells per side of that view (its largest world dimension)
    static constexpr int FULL_VIEW_CELLS = 0;
    // true = rotated sprites are scan-converted in a separate all-thread phase of the render kernel
    // instead of by the thread that owns the entity. Pays off where a frame mixes sprite kinds (a
    // warp then serialises a different long code path per lane): dodgeball and starpilot gain;
    // bossfight (all bullets alike) and the games with a rotated sprite or two lose.
    static constexpr bool DEFER_ROTATED = false;
    // true = the game has entities with render_z == -1 (drawn between the background and the grid
    // cells, draw_foreground basic-abstract-game.cpp:940): the frame is then composed in three steps
    static constexpr bool ENTS_BELOW_GRID = false;
    static PG_HD int image_for_type(Ctx &c, int type) { return type < 0 ? -type : type; }
    static PG_HD int theme_for_grid_obj(Ctx &c, int type) { return 0; }
    static PG_HD bool should_draw_entity(Ctx &c, int ei) { return true; }
    static PG_HD float get_tile_aspect_ratio(Ctx &c, int ei) { return 0; }
    static PG_HD void choose_center(Ctx &c, float &cx, float &cy) {
        cx = agent_of(c).x;
        cy = agent_of(c).y;
    }
    // returns true and rewrites r = {x, y, w, h} fractions when the sprite rect is adjusted
    static PG_HD bool get_adjusted_image_rect(Ctx &c, int type, double *adj) { return false; }
    static PG_HD bool should_preserve_type_themes(Ctx &c, int type) { return false; }
};

}  // namespace pg
