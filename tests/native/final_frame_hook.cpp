// TEST INFRASTRUCTURE — the reference never renders the state an episode ends in: Game::step (game.cpp:120-155)
// resets before it observes. This hook renders it for one env of a reference handle. It is compiled against the
// reference's own headers (read in place, like oracle/build_ref.py does) into a library of its own that links
// oracle/_ref/libenv_ref.so, so it works on the VecGame objects that library creates (tests/final_obs_oracle.py).
//
// The env takes `action` and replays game.cpp:121-142, everything before the reset decision (total_reward is
// private and not drawn, so it is left alone), then renders as Game::observe does (game.cpp:158-159) into
// rgb_out [64][64][3]. Returns why the level ends in this step, in the order of game.cpp:134: 1 the game ended it,
// 2 the time limit, 3 action -1; 0 when the step would not reset. It changes the env's state, so tests call it on
// a scratch handle, and only after libenv_observe, when no stepping thread owns the games.
#include "game.h"
#include "vecgame.h"

extern "C" __attribute__((visibility("default"))) int final_frame_hook(void *handle, int env, int action, uint8_t *rgb_out) {
    Game &g = *((VecGame *)handle)->games[env];
    g.action = action;
    g.cur_time += 1;
    bool force = false;
    if (g.action == -1) {
        g.action = g.default_action;
        force = true;
    }
    g.step_data.reward = 0;
    g.step_data.done = false;
    g.step_data.level_complete = false;
    g.game_step();
    const int cause = g.step_data.done ? 1 : (g.cur_time >= g.timeout ? 2 : (force ? 3 : 0));
    g.step_data.done = g.step_data.done || force || (g.cur_time >= g.timeout);
    if (g.step_data.reward != 0) {
        g.last_reward_timer = 10;
        g.last_reward = g.step_data.reward;
    }
    g.prev_level_seed = g.current_level_seed;
    g.render_to_buf(g.render_buf, RES_W, RES_H, false);
    bgr32_to_rgb888(rgb_out, g.render_buf, RES_W, RES_H);
    return cause;
}
