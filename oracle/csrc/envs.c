/* Scalar plain-C restatement of oracle/SPEC.md (breakout, snake, pong) + the reference vectoriser's send loop.
 * TEST INFRASTRUCTURE (see oracle/__init__.py): the checker for the CUDA env kernels and the CPU baseline.
 *
 * Vectoriser semantics follow reference pufferlib/vector.py:137-156 (per env: `if env.done: reset() else
 * step()`), emulation.py:187-192,219-224 (buffer rows) and postprocess.py:22-54 (EpisodeStats).  The dynamics
 * are OUR spec (parity unpinned against the reference, SPEC.md header).  One env at a time, straightforward
 * array code -- deliberately not shaped like the CUDA kernels.  `#pragma omp parallel for` over envs is the
 * "all host threads" CPU baseline; envs are independent so results do not depend on the thread count.
 */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#ifdef _OPENMP
#include <omp.h>
#endif

enum { K_BREAKOUT = 1, K_SNAKE = 2, K_PONG = 3 };

static uint32_t mix32(uint64_t x) {
    x += 0x9E3779B97F4A7C15ull;
    x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
    x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
    x ^= x >> 31;
    return (uint32_t)(x >> 32);
}

typedef struct {
    uint64_t seed;
    uint32_t ctr;
    int done;
    double ep_return;
    int ep_length;
    /* breakout */
    int px, bx, by, vx, vy, in_play, wait, lives, tick, bricks_left;
    uint8_t bricks[120];
    /* snake */
    int head, dir, len;
    uint8_t* grid;       /* [256], allocated for snake only */
    /* pong */
    int ly, ry, score_l, score_r;
    uint8_t (*frames)[84 * 84];  /* [4][7056], allocated for pong only */
} Env;

typedef struct {
    int kind, n;
    int iparam[8];
    int64_t offset;
    Env* envs;
    uint8_t* ext;   /* kind-specific per-env storage */
} Vec;

static uint32_t draw(Env* e) {
    uint32_t r = mix32(e->seed * 0x9E3779B97F4A7C15ull + (uint64_t)e->ctr * 0xD1B54A32D192ED03ull);
    e->ctr += 1;
    return r;
}

/* ------------------------------------------------------------------ breakout */
static void breakout_ball_on_paddle(Env* e) { e->bx = e->px + 11; e->by = 188; e->vx = 0; e->vy = 0; }

static void breakout_reset(Env* e) {
    e->px = 68; e->lives = 5; e->tick = 0; e->in_play = 0; e->wait = 0; e->bricks_left = 120;
    memset(e->bricks, 1, 120);
    breakout_ball_on_paddle(e);
}

static float breakout_step(Env* e, int a, int max_ticks, int* terminal, float* score) {
    static const int LAUNCH_VX[4] = {-2, -1, 1, 2};
    static const int HIT_VX[6] = {-3, -2, -1, 1, 2, 3};
    int reward = 0;
    if (a == 2) { e->px += 4; if (e->px > 136) e->px = 136; }
    if (a == 3) { e->px -= 4; if (e->px < 0) e->px = 0; }
    if (!e->in_play) {
        e->wait += 1;
        e->bx = e->px + 11; e->by = 188;
        if (a == 1 || e->wait >= 16) { e->in_play = 1; e->vy = -2; e->vx = LAUNCH_VX[draw(e) & 3]; }
    } else {
        e->bx += e->vx; e->by += e->vy;
        if (e->bx < 0) { e->bx = -e->bx; e->vx = -e->vx; }
        if (e->bx > 158) { e->bx = 316 - e->bx; e->vx = -e->vx; }
        if (e->by < 0) { e->by = -e->by; e->vy = -e->vy; }
        int cx = e->bx + 1, cy = e->by + 1;
        if (cy >= 30 && cy < 66) {
            int row = (cy - 30) / 6, col = cx / 8;
            if (e->bricks[row * 20 + col]) {
                e->bricks[row * 20 + col] = 0;
                e->bricks_left -= 1;
                reward += row < 2 ? 7 : (row < 4 ? 4 : 1);
                e->vy = -e->vy;
            }
        }
        if (e->vy > 0 && e->by >= 188 && e->by <= 192 && e->bx + 2 > e->px && e->bx < e->px + 24) {
            int off = e->bx + 1 - e->px;
            if (off < 0) off = 0;
            if (off > 23) off = 23;
            e->vy = -2; e->by = 188; e->vx = HIT_VX[off / 4];
        } else if (e->by >= 198) {
            e->lives -= 1; e->in_play = 0; e->wait = 0;
            breakout_ball_on_paddle(e);
        }
    }
    e->tick += 1;
    *terminal = (e->lives == 0 || e->bricks_left == 0 || e->tick >= max_ticks);
    *score = (float)(120 - e->bricks_left) / 120.0f;
    return (float)reward;
}

static void breakout_obs(const Env* e, float* o) {
    o[0] = (float)e->px / 256.0f; o[1] = (float)e->bx / 256.0f; o[2] = (float)e->by / 256.0f;
    o[3] = (float)e->vx / 4.0f; o[4] = (float)e->vy / 4.0f; o[5] = (float)e->lives / 8.0f;
    o[6] = (float)e->in_play; o[7] = (float)e->bricks_left / 128.0f;
    for (int i = 0; i < 120; i++) o[8 + i] = (float)e->bricks[i];
}

/* ------------------------------------------------------------------ snake */
static void snake_place_food(Env* e, int num_empty) {
    int k = (int)(draw(e) % (uint32_t)num_empty);
    for (int c = 0; c < 256; c++) {
        if (e->grid[c] == 0) {
            if (k == 0) { e->grid[c] = 255; return; }
            k--;
        }
    }
}

static void snake_reset(Env* e) {
    memset(e->grid, 0, 256);
    e->head = 136; e->grid[136] = 254; e->grid[135] = 1;
    e->len = 2; e->dir = 3; e->tick = 0;
    snake_place_food(e, 254);
}

static float snake_step(Env* e, int a, int max_ticks, int* terminal, float* score) {
    static const int DX[4] = {0, 0, -1, 1}, DY[4] = {-1, 1, 0, 0};
    float reward = 0.f;
    int term = 0;
    if (a != (e->dir ^ 1)) e->dir = a;
    int x = e->head & 15, y = e->head >> 4;
    int nx = x + DX[e->dir], ny = y + DY[e->dir];
    int dead = nx < 0 || nx > 15 || ny < 0 || ny > 15;
    int nc = dead ? 0 : ny * 16 + nx;
    if (!dead) {
        int q = e->grid[nc];
        if (q >= 2 && q <= 250) dead = 1;
    }
    if (dead) {
        reward = -1.f; term = 1;
    } else {
        int eat = e->grid[nc] == 255;
        if (eat) { e->len += 1; reward = 1.f; }
        else {
            for (int c = 0; c < 256; c++)
                if (e->grid[c] >= 1 && e->grid[c] <= 250) e->grid[c] -= 1;
        }
        e->grid[e->head] = (uint8_t)(e->len - 1);
        e->grid[nc] = 254;
        e->head = nc;
        if (eat) {
            if (e->len >= 250) term = 1;
            else snake_place_food(e, 256 - e->len);
        }
    }
    e->tick += 1;
    if (e->tick >= max_ticks) term = 1;
    *terminal = term;
    *score = (float)(e->len - 2);
    return reward;
}

/* ------------------------------------------------------------------ pong */
static void pong_serve(Env* e) {
    uint32_t r = draw(e);
    e->bx = 41; e->by = 41;
    e->vx = (r & 1) ? 2 : -2;
    e->vy = (int)((r >> 1) % 5) - 2;
}

static void pong_render(const Env* e, uint8_t* f) {
    memset(f, 0, 84 * 84);
    for (int y = e->ly; y < e->ly + 12; y++) for (int x = 4; x < 6; x++) f[y * 84 + x] = 128;
    for (int y = e->ry; y < e->ry + 12; y++) for (int x = 78; x < 80; x++) f[y * 84 + x] = 192;
    for (int y = e->by; y < e->by + 2; y++)
        for (int x = e->bx; x < e->bx + 2; x++)
            if (x >= 0 && x < 84 && y >= 0 && y < 84) f[y * 84 + x] = 255;
}

static void pong_reset(Env* e) {
    e->ly = 36; e->ry = 36; e->score_l = 0; e->score_r = 0; e->tick = 0;
    pong_serve(e);
    pong_render(e, e->frames[3]);
    for (int s = 0; s < 3; s++) memcpy(e->frames[s], e->frames[3], 84 * 84);
}

static float pong_step(Env* e, int a, int max_score, int max_ticks, int* terminal, float* score) {
    float reward = 0.f;
    if (a == 2 || a == 4) { e->ry -= 3; if (e->ry < 0) e->ry = 0; }
    if (a == 3 || a == 5) { e->ry += 3; if (e->ry > 72) e->ry = 72; }
    int tgt = e->by - 5;
    if (tgt < 0) tgt = 0;
    if (tgt > 72) tgt = 72;
    if (e->ly < tgt) { e->ly += 2; if (e->ly > tgt) e->ly = tgt; }
    else if (e->ly > tgt) { e->ly -= 2; if (e->ly < tgt) e->ly = tgt; }
    e->bx += e->vx; e->by += e->vy;
    if (e->by < 0) { e->by = -e->by; e->vy = -e->vy; }
    if (e->by > 82) { e->by = 164 - e->by; e->vy = -e->vy; }
    if (e->vx > 0 && e->bx >= 76 && e->bx <= 78 && e->by + 2 > e->ry && e->by < e->ry + 12) {
        e->vx = -2; e->bx = 76; e->vy = (e->by + 1 - e->ry - 6) / 3;
    } else if (e->vx < 0 && e->bx >= 4 && e->bx <= 6 && e->by + 2 > e->ly && e->by < e->ly + 12) {
        e->vx = 2; e->bx = 6; e->vy = (e->by + 1 - e->ly - 6) / 3;
    }
    if (e->bx < 0) { e->score_r += 1; reward = 1.f; pong_serve(e); }
    else if (e->bx > 82) { e->score_l += 1; reward = -1.f; pong_serve(e); }
    e->tick += 1;
    *terminal = (e->score_l >= max_score || e->score_r >= max_score || e->tick >= max_ticks);
    *score = (float)(e->score_r - e->score_l);
    memmove(e->frames[0], e->frames[1], 3 * 84 * 84);
    pong_render(e, e->frames[3]);
    return reward;
}

/* ------------------------------------------------------------------ vectoriser */
static int obs_bytes_of(int kind) { return kind == K_BREAKOUT ? 512 : (kind == K_SNAKE ? 256 : 4 * 84 * 84); }

static int param(const Vec* v, int i, int dflt) { return v->iparam[i] > 0 ? v->iparam[i] : dflt; }

static void write_obs(const Vec* v, const Env* e, uint8_t* row) {
    if (v->kind == K_BREAKOUT) breakout_obs(e, (float*)row);
    else if (v->kind == K_SNAKE) memcpy(row, e->grid, 256);
    else memcpy(row, e->frames, 4 * 84 * 84);
}

static void reset_env(const Vec* v, Env* e) {
    if (v->kind == K_BREAKOUT) breakout_reset(e);
    else if (v->kind == K_SNAKE) snake_reset(e);
    else pong_reset(e);
    e->done = 0; e->ep_return = 0.0; e->ep_length = 0;
}

void* oracle_vec_create(int kind, int n, int64_t env_index_offset, const int* iparam) {
    if (kind < K_BREAKOUT || kind > K_PONG || n < 1) return NULL;
    Vec* v = (Vec*)calloc(1, sizeof(Vec));
    v->kind = kind; v->n = n; v->offset = env_index_offset;
    if (iparam) memcpy(v->iparam, iparam, sizeof(v->iparam));
    v->envs = (Env*)calloc((size_t)n, sizeof(Env));
    const size_t ext = kind == K_SNAKE ? 256 : (kind == K_PONG ? 4 * 84 * 84 : 0);
    if (ext) v->ext = (uint8_t*)calloc((size_t)n, ext);
    for (int i = 0; i < n; i++) {
        v->envs[i].done = 1;
        if (kind == K_SNAKE) v->envs[i].grid = v->ext + (size_t)i * ext;
        if (kind == K_PONG) v->envs[i].frames = (uint8_t (*)[84 * 84])(v->ext + (size_t)i * ext);
    }
    return v;
}

void oracle_vec_destroy(void* h) {
    Vec* v = (Vec*)h;
    if (!v) return;
    free(v->envs);
    free(v->ext);
    free(v);
}

int oracle_vec_obs_bytes(void* h) { return obs_bytes_of(((Vec*)h)->kind); }

void oracle_set_threads(int n) {
#ifdef _OPENMP
    if (n > 0) omp_set_num_threads(n);
#else
    (void)n;
#endif
}

int oracle_max_threads(void) {
#ifdef _OPENMP
    return omp_get_max_threads();
#else
    return 1;
#endif
}

/* vector.py:112-135: env i <- seed + (offset + i), reset, reset rows */
void oracle_vec_reset(void* h, uint64_t seed, uint8_t* obs, float* rewards, uint8_t* terminals,
                      uint8_t* truncations, uint8_t* masks) {
    Vec* v = (Vec*)h;
    const int ob = obs_bytes_of(v->kind);
#pragma omp parallel for schedule(static)
    for (int i = 0; i < v->n; i++) {
        Env* e = &v->envs[i];
        e->seed = seed + (uint64_t)(v->offset + i);
        e->ctr = 0;
        reset_env(v, e);
        write_obs(v, e, obs + (size_t)i * ob);
        rewards[i] = 0.f; terminals[i] = 0; truncations[i] = 0; masks[i] = 1;
    }
}

/* vector.py:137-156.  info_* are valid where terminals[i] != 0 (EpisodeStats, postprocess.py:36-52). */
void oracle_vec_step(void* h, const int64_t* actions, uint8_t* obs, float* rewards, uint8_t* terminals,
                     uint8_t* truncations, uint8_t* masks, double* info_return, int* info_length,
                     float* info_score) {
    Vec* v = (Vec*)h;
    const int ob = obs_bytes_of(v->kind);
#pragma omp parallel for schedule(static)
    for (int i = 0; i < v->n; i++) {
        Env* e = &v->envs[i];
        float reward = 0.f, score = 0.f;
        int term = 0;
        if (e->done) {
            reset_env(v, e);
        } else {
            int a = (int)actions[i];
            if (v->kind == K_BREAKOUT) reward = breakout_step(e, a, param(v, 0, 4096), &term, &score);
            else if (v->kind == K_SNAKE) reward = snake_step(e, a, param(v, 0, 1024), &term, &score);
            else reward = pong_step(e, a, param(v, 0, 5), param(v, 1, 4096), &term, &score);
            e->ep_return += (double)reward;
            e->ep_length += 1;
            e->done = term;
            if (term) {
                if (info_return) info_return[i] = e->ep_return;
                if (info_length) info_length[i] = e->ep_length;
                if (info_score) info_score[i] = score;
            }
        }
        write_obs(v, e, obs + (size_t)i * ob);
        rewards[i] = reward; terminals[i] = (uint8_t)term; truncations[i] = 0; masks[i] = 1;
    }
}
