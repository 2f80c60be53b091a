/* Scalar plain-C restatement of oracle/SPEC_PONG_VERSUS.md (two-player pong from pixels) + the reference vectoriser's
 * send loop over a PettingZoo env with two agents.
 * TEST INFRASTRUCTURE (see oracle/__init__.py): the checker for the pong_versus CUDA kernel.
 *
 * Vectoriser semantics follow reference pufferlib/vector.py:97-110,137-156 (agent a of env e at row e*2 + a; per env:
 * `if env.done: reset() else step()`), emulation.py:236-420 (PettingZooPufferEnv: reset rows r=0, terminal=False;
 * done = all agents terminal).  The frame stack keeps S frames the way gymnasium's FrameStack does (every slot the
 * first frame on a reset; drop the oldest, append the newest on a step).  One env at a time; each agent's frame is
 * drawn from that agent's side of the field directly -- deliberately not shaped like the CUDA kernel, which renders
 * from pong's state with a seat argument.
 */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define PV_FRAME (84 * 84)

typedef struct {
    uint64_t seed;
    uint32_t ctr;
    int done;
    int ly, ry, bx, by, vx, vy, score_l, score_r, tick;
} PvEnv;

typedef struct {
    int n, S, max_score, max_ticks;
    int64_t offset;
    PvEnv* envs;
} PvVec;

static uint32_t pv_mix32(uint64_t x) {
    x += 0x9E3779B97F4A7C15ull;
    x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
    x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
    x ^= x >> 31;
    return (uint32_t)(x >> 32);
}

static void pv_serve(PvEnv* e) {
    uint32_t r = pv_mix32(e->seed * 0x9E3779B97F4A7C15ull + (uint64_t)e->ctr * 0xD1B54A32D192ED03ull);
    e->ctr += 1;
    e->bx = 41; e->by = 41;
    e->vx = (r & 1) ? 2 : -2;
    e->vy = (int)((r >> 1) % 5) - 2;
}

static void pv_reset(PvEnv* e) {
    e->ly = 36; e->ry = 36; e->score_l = 0; e->score_r = 0; e->tick = 0;
    pv_serve(e);
}

static int pv_move(int y, int a) {
    if (a == 2 || a == 4) { y -= 3; if (y < 0) y = 0; }
    if (a == 3 || a == 5) { y += 3; if (y > 72) y = 72; }
    return y;
}

/* one step from both actions; returns agent 0's reward */
static float pv_step(PvEnv* e, int a0, int a1, int max_score, int max_ticks, int* terminal) {
    float reward = 0.f;
    e->ry = pv_move(e->ry, a0);   /* agent 0: the right paddle */
    e->ly = pv_move(e->ly, a1);   /* agent 1: the left paddle */
    e->bx += e->vx; e->by += e->vy;
    if (e->by < 0) { e->by = -e->by; e->vy = -e->vy; }
    if (e->by > 82) { e->by = 164 - e->by; e->vy = -e->vy; }
    if (e->vx > 0 && e->bx >= 76 && e->bx <= 78 && e->by + 2 > e->ry && e->by < e->ry + 12) {
        e->vx = -2; e->bx = 76; e->vy = (e->by + 1 - e->ry - 6) / 3;
    } else if (e->vx < 0 && e->bx >= 4 && e->bx <= 6 && e->by + 2 > e->ly && e->by < e->ly + 12) {
        e->vx = 2; e->bx = 6; e->vy = (e->by + 1 - e->ly - 6) / 3;
    }
    if (e->bx < 0) { e->score_r += 1; reward = 1.f; pv_serve(e); }
    else if (e->bx > 82) { e->score_l += 1; reward = -1.f; pv_serve(e); }
    e->tick += 1;
    *terminal = (e->score_l >= max_score || e->score_r >= max_score || e->tick >= max_ticks);
    return reward;
}

/* agent a's view: its own paddle at x = 78..79 (192), the other's at x = 4..5 (128), the ball (255) drawn last;
 * agent 1 stands on the left, so for it field column c is frame column 83 - c */
static void pv_render(const PvEnv* e, int agent, uint8_t* f) {
    const int own = agent == 0 ? e->ry : e->ly, opp = agent == 0 ? e->ly : e->ry;
    memset(f, 0, PV_FRAME);
    for (int y = opp; y < opp + 12; y++) for (int x = 4; x < 6; x++) f[y * 84 + x] = 128;
    for (int y = own; y < own + 12; y++) for (int x = 78; x < 80; x++) f[y * 84 + x] = 192;
    for (int y = e->by; y < e->by + 2; y++)
        for (int fx = e->bx; fx < e->bx + 2; fx++) {
            const int x = agent == 0 ? fx : 83 - fx;
            if (x >= 0 && x < 84 && y >= 0 && y < 84) f[y * 84 + x] = 255;
        }
}

/* obs row of agent a of env i: S frames, oldest first */
static uint8_t* pv_row(const PvVec* v, uint8_t* obs, int i, int a) {
    return obs + ((size_t)i * 2 + (size_t)a) * (size_t)v->S * PV_FRAME;
}

static void pv_fill(const PvVec* v, const PvEnv* e, uint8_t* obs, int i) {
    for (int a = 0; a < 2; a++) {
        uint8_t* row = pv_row(v, obs, i, a);
        pv_render(e, a, row);
        for (int s = 1; s < v->S; s++) memcpy(row + (size_t)s * PV_FRAME, row, PV_FRAME);
    }
}

static void pv_push(const PvVec* v, const PvEnv* e, uint8_t* obs, int i) {
    for (int a = 0; a < 2; a++) {
        uint8_t* row = pv_row(v, obs, i, a);
        memmove(row, row + PV_FRAME, (size_t)(v->S - 1) * PV_FRAME);
        pv_render(e, a, row + (size_t)(v->S - 1) * PV_FRAME);
    }
}

void* oracle_pv_create(int n, int64_t env_index_offset, int framestack, int max_score, int max_ticks) {
    if (n < 1 || (framestack != 1 && framestack != 4)) return NULL;
    PvVec* v = (PvVec*)calloc(1, sizeof(PvVec));
    v->n = n; v->S = framestack; v->offset = env_index_offset;
    v->max_score = max_score > 0 ? max_score : 5;
    v->max_ticks = max_ticks > 0 ? max_ticks : 4096;
    v->envs = (PvEnv*)calloc((size_t)n, sizeof(PvEnv));
    for (int i = 0; i < n; i++) v->envs[i].done = 1;
    return v;
}

void oracle_pv_destroy(void* h) {
    PvVec* v = (PvVec*)h;
    if (!v) return;
    free(v->envs);
    free(v);
}

/* vector.py:112-135: env i <- seed + (offset + i), reset, reset rows for both agents */
void oracle_pv_reset(void* h, uint64_t seed, uint8_t* obs, float* rewards, uint8_t* terminals) {
    PvVec* v = (PvVec*)h;
    for (int i = 0; i < v->n; i++) {
        PvEnv* e = &v->envs[i];
        e->seed = seed + (uint64_t)(v->offset + i);
        e->ctr = 0;
        pv_reset(e);
        e->done = 0;
        pv_fill(v, e, obs, i);
        rewards[2 * i] = rewards[2 * i + 1] = 0.f;
        terminals[2 * i] = terminals[2 * i + 1] = 0;
    }
}

/* vector.py:137-156 over 2n agent rows.  info_score (agent 0's score) / info_length are valid where env i's rows are
 * terminal. */
void oracle_pv_step(void* h, const int64_t* actions, uint8_t* obs, float* rewards, uint8_t* terminals,
                    int* info_score, int* info_length) {
    PvVec* v = (PvVec*)h;
    for (int i = 0; i < v->n; i++) {
        PvEnv* e = &v->envs[i];
        float r0 = 0.f, r1 = 0.f;
        int term = 0;
        if (e->done) {
            pv_reset(e);           /* the draw counter runs on across resets */
            e->done = 0;
            pv_fill(v, e, obs, i);
        } else {
            r0 = pv_step(e, (int)actions[2 * i], (int)actions[2 * i + 1], v->max_score, v->max_ticks, &term);
            r1 = r0 == 0.f ? 0.f : -r0;
            e->done = term;
            pv_push(v, e, obs, i);
            if (term) {
                info_score[i] = e->score_r - e->score_l;
                info_length[i] = e->tick;
            }
        }
        rewards[2 * i] = r0; rewards[2 * i + 1] = r1;
        terminals[2 * i] = terminals[2 * i + 1] = (uint8_t)term;
    }
}
