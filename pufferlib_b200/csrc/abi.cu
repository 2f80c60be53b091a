// abi.cu -- C-ABI plumbing of libpuffer_b200.so: error strings, env handle lifecycle and dispatch.
#include <stdarg.h>
#include <stdlib.h>
#include <string.h>

#include "env_common.cuh"
#include "frame_stack.cuh"

static thread_local char g_err[512] = "";

void pb_set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

unsigned long long g_pb_launches = 0;

extern "C" const char* pb_last_error(void) { return g_err; }
extern "C" uint64_t pb_launch_count(void) { return g_pb_launches; }
extern "C" int pb_abi_version(void) { return PB_ABI_VERSION; }

extern "C" int pb_device_count(int* out_count) {
    PB_REQUIRE(out_count, PB_ERR_INVALID, "pb_device_count: null pointer");
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess) {
        pb_set_error("cudaGetDeviceCount: %s", cudaGetErrorString(e));
        *out_count = 0;
        return PB_ERR_CUDA;
    }
    *out_count = n;
    return PB_OK;
}

int pb_env_alloc_common(pb_env* env) {
    const size_t n = (size_t)env->cfg.num_envs;
    PB_CUDA(cudaMalloc(&env->d_done, n));
    PB_CUDA(cudaMalloc(&env->d_ep_return, n * sizeof(double)));
    PB_CUDA(cudaMalloc(&env->d_ep_length, n * sizeof(int32_t)));
    PB_CUDA(cudaMalloc(&env->d_row_return, n * sizeof(double)));
    PB_CUDA(cudaMalloc(&env->d_row_length, n * sizeof(int32_t)));
    PB_CUDA(cudaMalloc(&env->d_row_score, n * sizeof(float)));
    PB_CUDA(cudaMalloc(&env->d_stats, PB_STAT_SLOTS * 4 * sizeof(double)));
    PB_CUDA(cudaMallocHost(&env->h_stats_pinned, PB_STAT_SLOTS * 4 * sizeof(double)));
    PB_CUDA(cudaMemset(env->d_done, 1, n));  // GymnasiumPufferEnv starts with done = True (emulation.py:129)
    PB_CUDA(cudaMemset(env->d_ep_return, 0, n * sizeof(double)));
    PB_CUDA(cudaMemset(env->d_ep_length, 0, n * sizeof(int32_t)));
    PB_CUDA(cudaMemset(env->d_row_return, 0, n * sizeof(double)));
    PB_CUDA(cudaMemset(env->d_row_length, 0, n * sizeof(int32_t)));
    PB_CUDA(cudaMemset(env->d_row_score, 0, n * sizeof(float)));
    PB_CUDA(cudaMemset(env->d_stats, 0, PB_STAT_SLOTS * 4 * sizeof(double)));
    return PB_OK;
}

void pb_env_free_common(pb_env* env) {
    cudaFree(env->d_done);
    cudaFree(env->d_ep_return);
    cudaFree(env->d_ep_length);
    cudaFree(env->d_row_return);
    cudaFree(env->d_row_length);
    cudaFree(env->d_row_score);
    cudaFree(env->d_stats);
    if (env->h_stats_pinned) cudaFreeHost(env->h_stats_pinned);
}

extern "C" int pb_env_create_ex(const pb_env_config* cfg, const double* dparam_host, int32_t n_dparam, pb_env** out) {
    PB_REQUIRE(cfg && out, PB_ERR_INVALID, "pb_env_create: null pointer");
    PB_REQUIRE(n_dparam >= 0 && (n_dparam == 0 || dparam_host), PB_ERR_INVALID, "pb_env_create_ex: bad dparam");
    *out = nullptr;
    PB_REQUIRE(cfg->num_envs >= 1, PB_ERR_INVALID, "num_envs must be at least 1");  // vector.py:578-579
    PB_REQUIRE(cfg->kind >= PB_ENV_SQUARED && cfg->kind <= PB_ENV_PONG_VERSUS, PB_ERR_INVALID, "unknown env kind %d",
               cfg->kind);
    if (cfg->kind == PB_ENV_PONG || cfg->kind == PB_ENV_BREAKOUT_PIXELS) {
        const int rc = fs_pre_check(cfg);   // the Atari preprocessing options, refused before anything is allocated
        if (rc != PB_OK) return rc;
    }
    if (cfg->kind == PB_ENV_PONG_VERSUS) {
        const int rc = pb_pong_versus_check(cfg);
        if (rc != PB_OK) return rc;
    }
    int ndev = 0;
    PB_CUDA(cudaGetDeviceCount(&ndev));
    PB_REQUIRE(cfg->device >= 0 && cfg->device < ndev, PB_ERR_CUDA, "CUDA device %d not available (%d devices)",
               cfg->device, ndev);
    PB_CUDA(cudaSetDevice(cfg->device));
    pb_env* env = (pb_env*)calloc(1, sizeof(pb_env));
    PB_REQUIRE(env, PB_ERR_CUDA, "out of host memory");
    env->cfg = *cfg;
    env->agents_per_env = 1;
    int rc = pb_env_alloc_common(env);
    if (rc == PB_OK) {
        switch (cfg->kind) {
            case PB_ENV_SQUARED: rc = pb_squared_create(env); break;
            case PB_ENV_BREAKOUT: rc = pb_breakout_create(env); break;
            case PB_ENV_SNAKE: rc = pb_snake_create(env); break;
            case PB_ENV_PONG: rc = pb_pong_create(env); break;
            case PB_ENV_BREAKOUT_PIXELS: rc = pb_breakout_pixels_create(env); break;
            case PB_ENV_PONG_VERSUS: rc = pb_pong_versus_create(env); break;
            default: rc = pb_ocean_create(env, dparam_host, n_dparam); break;
        }
    }
    if (rc != PB_OK) {
        if (env->vt && env->vt->destroy) env->vt->destroy(env);
        pb_env_free_common(env);
        free(env);
        return rc;
    }
    env->info.num_envs = cfg->num_envs;
    *out = env;
    return PB_OK;
}

extern "C" int pb_env_create(const pb_env_config* cfg, pb_env** out) {
    return pb_env_create_ex(cfg, nullptr, 0, out);
}

extern "C" int pb_env_destroy(pb_env* env) {
    if (!env) return PB_OK;
    cudaSetDevice(env->cfg.device);
    if (env->vt && env->vt->destroy) env->vt->destroy(env);
    pb_env_free_common(env);
    free(env);
    return PB_OK;
}

extern "C" int pb_env_get_info(const pb_env* env, pb_env_info* out) {
    PB_REQUIRE(env && out, PB_ERR_INVALID, "pb_env_get_info: null pointer");
    *out = env->info;
    return PB_OK;
}

extern "C" int pb_env_agents_per_env(const pb_env* env, int32_t* out) {
    PB_REQUIRE(env && out, PB_ERR_INVALID, "pb_env_agents_per_env: null pointer");
    *out = env->agents_per_env;
    return PB_OK;
}

static int check_out(const pb_env* env, const pb_env_out* out, const char* who) {
    PB_REQUIRE(out && out->obs && out->rewards && out->terminals && out->truncations && out->masks, PB_ERR_INVALID,
               "%s: obs/rewards/terminals/truncations/masks pointers are required", who);
    PB_REQUIRE(out->obs_stride >= env->info.obs_bytes, PB_ERR_INVALID, "%s: obs_stride %lld < obs_bytes %lld", who,
               (long long)out->obs_stride, (long long)env->info.obs_bytes);
    return PB_OK;
}

extern "C" int pb_env_reset(pb_env* env, uint64_t seed, const pb_env_out* out, void* stream) {
    PB_REQUIRE(env, PB_ERR_INVALID, "pb_env_reset: null handle");
    int rc = check_out(env, out, "pb_env_reset");
    if (rc) return rc;
    PB_CUDA(cudaSetDevice(env->cfg.device));
    env->write_const = true;
    rc = env->vt->reset(env, seed, out, (cudaStream_t)stream);
    if (rc == PB_OK) {
        env->was_reset = true;
        env->const_trunc = out->truncations;
        env->const_masks = out->masks;
        env->cur_obs = out->obs;
        env->cur_obs_stride = out->obs_stride;
    }
    return rc;
}

extern "C" int pb_env_step(pb_env* env, const int64_t* actions, const pb_env_out* out, void* stream) {
    PB_REQUIRE(env, PB_ERR_INVALID, "pb_env_step: null handle");
    PB_REQUIRE(env->was_reset, PB_ERR_STATE, "step() called before reset()");  // emulation.py:198-199
    PB_REQUIRE(actions, PB_ERR_INVALID, "pb_env_step: null actions");
    int rc = check_out(env, out, "pb_env_step");
    if (rc) return rc;
    PB_CUDA(cudaSetDevice(env->cfg.device));
    env->write_const = out->truncations != env->const_trunc || out->masks != env->const_masks;
    rc = env->vt->step(env, actions, out, (cudaStream_t)stream);
    if (rc == PB_OK) {
        env->const_trunc = out->truncations;
        env->const_masks = out->masks;
        env->cur_obs = out->obs;
        env->cur_obs_stride = out->obs_stride;
    }
    return rc;
}

extern "C" int pb_env_episode_rows(pb_env* env, const double** episode_return, const int32_t** episode_length,
                                   const float** score) {
    PB_REQUIRE(env, PB_ERR_INVALID, "pb_env_episode_rows: null handle");
    if (episode_return) *episode_return = env->d_row_return;
    if (episode_length) *episode_length = env->d_row_length;
    if (score) *score = env->d_row_score;
    return PB_OK;
}

extern "C" int pb_env_episode_score_f64(pb_env* env, const double** score) {
    PB_REQUIRE(env && score, PB_ERR_INVALID, "pb_env_episode_score_f64: null pointer");
    *score = env->d_row_score64;
    return PB_OK;
}

extern "C" int pb_env_game_ended(pb_env* env, const uint8_t** ended) {
    PB_REQUIRE(env && ended, PB_ERR_INVALID, "pb_env_game_ended: null pointer");
    *ended = env->d_ended;
    return PB_OK;
}

extern "C" int pb_env_stats_read(pb_env* env, double* out4_host, int clear, void* stream) {
    PB_REQUIRE(env && out4_host, PB_ERR_INVALID, "pb_env_stats_read: null pointer");
    cudaStream_t s = (cudaStream_t)stream;
    PB_CUDA(cudaSetDevice(env->cfg.device));
    const size_t bytes = PB_STAT_SLOTS * 4 * sizeof(double);
    PB_CUDA(cudaMemcpyAsync(env->h_stats_pinned, env->d_stats, bytes, cudaMemcpyDeviceToHost, s));
    if (clear) PB_CUDA(cudaMemsetAsync(env->d_stats, 0, bytes, s));
    PB_CUDA(cudaStreamSynchronize(s));
    for (int k = 0; k < 4; ++k) out4_host[k] = 0.0;
    for (int slot = 0; slot < PB_STAT_SLOTS; ++slot)
        for (int k = 0; k < 4; ++k) out4_host[k] += env->h_stats_pinned[slot * 4 + k];
    return PB_OK;
}

extern "C" int pb_env_agent_stats_read(pb_env* env, double* out4_host, int clear, void* stream) {
    PB_REQUIRE(env && out4_host, PB_ERR_INVALID, "pb_env_agent_stats_read: null pointer");
    PB_REQUIRE(env->d_agent_stats, PB_ERR_INVALID, "pb_env_agent_stats_read: env kind %d has one agent per env",
               env->cfg.kind);
    cudaStream_t s = (cudaStream_t)stream;
    PB_CUDA(cudaSetDevice(env->cfg.device));
    const size_t bytes = 4 * sizeof(unsigned long long);
    unsigned long long* h = (unsigned long long*)env->h_stats_pinned;   // 32 of its bytes
    PB_CUDA(cudaMemcpyAsync(h, env->d_agent_stats, bytes, cudaMemcpyDeviceToHost, s));
    if (clear) PB_CUDA(cudaMemsetAsync(env->d_agent_stats, 0, bytes, s));
    PB_CUDA(cudaStreamSynchronize(s));
    // integer sums in two's complement (a score sum may be negative): exact below 2**53 in magnitude
    for (int k = 0; k < 4; ++k) out4_host[k] = (double)(long long)h[k];
    return PB_OK;
}

// cudaDevAttrMultiProcessorCount of the current device, cached per device ordinal
int pb_num_sms() {
    static int cache[64] = {0};
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return 132;
    if (!cache[dev]) {
        int n = 0;
        if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n < 1) n = 132;
        cache[dev] = n;
    }
    return cache[dev];
}
