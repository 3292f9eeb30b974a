// maze_ref -- drives the reference's own hard-maze code (gpu_implementation/gym_tensorflow/maze/maze.h, included from the
// reference checkout at compile time, never copied) so that tests/golden/make_golden_maze.py can pin the device maze to
// it.  Built by __graft_entry__.build() with `g++ -O2 -ffp-contract=off` (no fast-math) into oracle/_ref/maze_ref.
//
//   maze_ref MAZE_FILE reset                 -> stdout: float32 obs[11] of the reset state
//   maze_ref MAZE_FILE step    < records     -> stdout: per record float32 [x, y, heading, speed, ang_vel, collide,
//                                               t, reward, obs[11]]  (19 floats)
//       record (stdin, float32 x 9): x, y, heading, speed, ang_vel, collide (0/1), t (steps taken), then the action
//       a0, a1; the hero's fields are set directly
//   maze_ref MAZE_FILE episode T < actions   -> stdout: per episode, per step the 19 floats above
//       actions (stdin, float32): n episodes of [T][2], open loop from the reset state
//
// One step is the reference GPU path's MazeEnvironment::step (gym_tensorflow/maze/tf_maze.cpp): interpret_outputs(
// float(a0) + 0.5, 0.5 + float(a1)), Update(), one more step taken, and the reward -distance_to_target() when the count
// reaches 400, otherwise 0.
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "maze.h"

static const int MAZE_STEPS = 400;

static void put(const float* v, size_t n) {
    if (fwrite(v, sizeof(float), n, stdout) != n) exit(3);
}

// one step of the environment `e`, whose hero is already set, with `t` steps taken so far; writes the 19 output floats
static void step_and_emit(maze::Environment& e, int& t, float a0, float a1) {
    e.interpret_outputs(float(a0) + 0.5, 0.5 + float(a1));
    e.Update();
    t += 1;
    const float reward = t >= MAZE_STEPS ? -e.distance_to_target() : 0.0f;
    float out[19];
    out[0] = e.hero.location.x;
    out[1] = e.hero.location.y;
    out[2] = e.hero.heading;
    out[3] = e.hero.speed;
    out[4] = e.hero.ang_vel;
    out[5] = e.hero.collide ? 1.0f : 0.0f;
    out[6] = (float)t;
    out[7] = reward;
    e.generate_neural_inputs(out + 8);
    put(out, 19);
}

int main(int argc, char** argv) {
    if (argc < 3) {
        fprintf(stderr, "usage: maze_ref MAZE_FILE reset|step|episode T\n");
        return 2;
    }
    std::cout.rdbuf(std::cerr.rdbuf());        // the maze code's diagnostics ("NAN in inputs", ...) stay off the data
    maze::Environment e(argv[1]);
    if (e.get_sensor_size() != 11) return 4;
    if (!strcmp(argv[2], "reset")) {
        e.reset();
        float obs[11];
        e.generate_neural_inputs(obs);
        put(obs, 11);
    } else if (!strcmp(argv[2], "step")) {
        float r[9];
        while (fread(r, sizeof(float), 9, stdin) == 9) {
            e.reset();
            e.hero.location.x = r[0];
            e.hero.location.y = r[1];
            e.hero.heading = r[2];
            e.hero.speed = r[3];
            e.hero.ang_vel = r[4];
            e.hero.collide = r[5] != 0.0f;
            int t = (int)r[6];
            step_and_emit(e, t, r[7], r[8]);
        }
    } else if (!strcmp(argv[2], "episode") && argc == 4) {
        const int T = atoi(argv[3]);
        std::vector<float> a(2 * (size_t)T);
        while (fread(a.data(), sizeof(float), a.size(), stdin) == a.size()) {
            e.reset();
            int t = 0;
            for (int k = 0; k < T; ++k) step_and_emit(e, t, a[2 * k], a[2 * k + 1]);
        }
    } else {
        return 2;
    }
    return fflush(stdout) == 0 ? 0 : 3;
}
