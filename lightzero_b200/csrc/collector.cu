// collector.cu -- device-resident collector state (SURVEY 8(f) row f-3): the per-environment observation frame stacks the
// reference keeps in GameSegment.obs_segment / get_obs (lzero/mcts/buffer/game_segment.py:140-156, seeded with frame_stack_num
// copies of the first frame by the collector, lzero/worker/muzero_collector.py:451-457, one frame appended per step, :520-545,
// :640-700) and the search statistics GameSegment.store_search_stats appends after every search (game_segment.py:241-263).
// HBM-bound byte moves: each kernel touches every byte once with 16-byte accesses.
#include <string.h>

#include <algorithm>

#include "lz_common.cuh"

struct lz_frames {
    int B, stack, frame_bytes;      // frame_bytes = H * W (one uint8 channel per frame), a multiple of 16
    uint8_t *buf[2];                // ping-pong [B][stack][frame_bytes], oldest frame first
    int cur;                        // buf[cur] holds the current stacks
    uint8_t *d_new;                 // upload staging [B][frame_bytes]
    uint8_t *d_reset;               // upload staging [B]
};

struct lz_segments {
    int B, T, A;
    float *child_visits;            // [B][T][A]  visit_count / sum(visit_counts) per position of the root's legal list, 0 beyond it
    float *root_values;             // [B][T]
    int32_t *len;                   // [B] entries stored so far (<= T)
    float *improved_policy;         // [B][T][A] Gumbel MuZero improved policy by action id; allocated by the first store
};

namespace lz {

// out[b][k] = reset[b] ? new[b] : (k + 1 < stack ? in[b][k + 1] : new[b])      (uint4 = 16 frames bytes per thread)
__global__ void __launch_bounds__(256) k_frames_push(const uint4 *__restrict__ in, uint4 *__restrict__ out, const uint4 *__restrict__ nw,
                                                     const uint8_t *__restrict__ reset, int B, int stack, int fq)
{
    const size_t n = (size_t)B * stack * fq;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const int q = (int)(i % fq), k = (int)((i / fq) % stack), b = (int)(i / ((size_t)fq * stack));
        const bool rs = reset && reset[b];
        out[i] = (rs || k + 1 == stack) ? nw[(size_t)b * fq + q] : in[i + fq];
    }
}

// GameSegment.store_search_stats (game_segment.py:241-263), idx is None: one warp per environment
__global__ void __launch_bounds__(128) k_segments_store(const int32_t *__restrict__ visits, const float *__restrict__ values,
                                                        const uint8_t *__restrict__ active, float *child_visits, float *root_values,
                                                        int32_t *len, int B, int T, int A)
{
    const int b = blockIdx.x * 4 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (b >= B || (active && !active[b])) return;
    const int t = len[b];
    if (t >= T) return;                       // segment full: the host pads over / resets it (game_segment.py:183-224)
    long long sum = 0;
    for (int a = lane; a < A; a += 32) {
        const int v = visits[(size_t)b * A + a];
        if (v > 0) sum += v;                  // -1 marks positions beyond the legal list (lz_tree_results)
    }
    for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
    // Python: visit_count / sum_visits in float64 (sum_visits = 1e-6 when every count is 0), stored as float32 targets later
    const double denom = sum == 0 ? 1e-6 : (double)sum;
    for (int a = lane; a < A; a += 32) {
        const int v = visits[(size_t)b * A + a];
        child_visits[((size_t)b * T + t) * A + a] = v > 0 ? (float)((double)v / denom) : 0.0f;
    }
    if (lane == 0) {
        root_values[(size_t)b * T + t] = values[b];
        len[b] = t + 1;
    }
}

// GameSegment.store_search_stats(..., improved_policy=...) (game_segment.py:258-259): the improved policy goes in at the position
// len that k_segments_store then fills and advances past, under the same full-segment rule
__global__ void __launch_bounds__(128) k_segments_store_policy(const float *__restrict__ policy, const uint8_t *__restrict__ active,
                                                               float *improved_policy, const int32_t *len, int B, int T, int A)
{
    const int b = blockIdx.x * 4 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (b >= B || (active && !active[b])) return;
    const int t = len[b];
    if (t >= T) return;
    for (int a = lane; a < A; a += 32) improved_policy[((size_t)b * T + t) * A + a] = policy[(size_t)b * A + a];
}

// zeroes the `row` floats of every done segment b (all of them when done is null)
__global__ void k_segments_clear_rows(float *x, const uint8_t *__restrict__ done, int B, size_t row)
{
    const size_t n = (size_t)B * row;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
        if (!done || done[i / row]) x[i] = 0.0f;
}

__global__ void k_segments_reset(int32_t *len, const uint8_t *__restrict__ done, int B)
{
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b < B && (!done || done[b])) len[b] = 0;
}

}  // namespace lz

using namespace lz;

extern "C" {

int lz_frames_create(int B, int stack, int H, int W, lz_frames **out)
{
    LZ_REQUIRE(out && B > 0 && stack > 0 && H > 0 && W > 0, LZ_EINVAL, "lz_frames_create: bad argument");
    LZ_REQUIRE((H * W) % 16 == 0, LZ_EINVAL, "lz_frames_create: H * W = %d is not a multiple of 16", H * W);
    lz_frames *f = new lz_frames();
    memset(f, 0, sizeof(*f));
    f->B = B; f->stack = stack; f->frame_bytes = H * W;
    const size_t n = (size_t)B * stack * f->frame_bytes;
    int rc = dev_alloc(&f->buf[0], n);
    if (rc == LZ_OK) rc = dev_alloc(&f->buf[1], n);
    if (rc == LZ_OK) rc = dev_alloc(&f->d_new, (size_t)B * f->frame_bytes);
    if (rc == LZ_OK) rc = dev_alloc(&f->d_reset, (size_t)B);
    if (rc == LZ_OK) rc = setup_memset(f->buf[0], n);
    if (rc != LZ_OK) { lz_frames_destroy(f); return rc; }
    *out = f;
    return LZ_OK;
}

int lz_frames_destroy(lz_frames *f)
{
    if (!f) return LZ_OK;
    cudaFree(f->buf[0]); cudaFree(f->buf[1]); cudaFree(f->d_new); cudaFree(f->d_reset);
    delete f;
    return LZ_OK;
}

int lz_frames_push(lz_frames *f, const uint8_t *d_new_frames, const uint8_t *d_reset, lz_stream s)
{
    LZ_REQUIRE(f && d_new_frames, LZ_EINVAL, "lz_frames_push: null argument");
    const int fq = f->frame_bytes / 16;
    const size_t n = (size_t)f->B * f->stack * fq;
    const int blocks = (int)((n + 255) / 256 < (size_t)kNumSMs * 8 ? (n + 255) / 256 : (size_t)kNumSMs * 8);
    k_frames_push<<<blocks, 256, 0, (cudaStream_t)s>>>(reinterpret_cast<const uint4 *>(f->buf[f->cur]), reinterpret_cast<uint4 *>(f->buf[f->cur ^ 1]),
                                                     reinterpret_cast<const uint4 *>(d_new_frames), d_reset, f->B, f->stack, fq);
    LZ_KERNEL_CHECK();
    f->cur ^= 1;
    return LZ_OK;
}

int lz_frames_push_host(lz_frames *f, const uint8_t *h_new_frames, const uint8_t *h_reset, lz_stream s)
{
    LZ_REQUIRE(f && h_new_frames, LZ_EINVAL, "lz_frames_push_host: null argument");
    LZ_CUDA_CHECK(cudaMemcpyAsync(f->d_new, h_new_frames, (size_t)f->B * f->frame_bytes, cudaMemcpyHostToDevice, (cudaStream_t)s));
    if (h_reset) LZ_CUDA_CHECK(cudaMemcpyAsync(f->d_reset, h_reset, (size_t)f->B, cudaMemcpyHostToDevice, (cudaStream_t)s));
    return lz_frames_push(f, f->d_new, h_reset ? f->d_reset : nullptr, s);
}

const uint8_t *lz_frames_stacked(lz_frames *f) { return f ? f->buf[f->cur] : nullptr; }

int lz_segments_create(int B, int T, int A, lz_segments **out)
{
    LZ_REQUIRE(out && B > 0 && T > 0 && A > 0, LZ_EINVAL, "lz_segments_create: bad argument");
    lz_segments *g = new lz_segments();
    memset(g, 0, sizeof(*g));
    g->B = B; g->T = T; g->A = A;
    int rc = dev_alloc(&g->child_visits, (size_t)B * T * A);
    if (rc == LZ_OK) rc = dev_alloc(&g->root_values, (size_t)B * T);
    if (rc == LZ_OK) rc = dev_alloc(&g->len, (size_t)B);
    if (rc == LZ_OK) rc = setup_memset(g->child_visits, (size_t)B * T * A * sizeof(float));
    if (rc == LZ_OK) rc = setup_memset(g->root_values, (size_t)B * T * sizeof(float));
    if (rc == LZ_OK) rc = setup_memset(g->len, (size_t)B * sizeof(int32_t));
    if (rc != LZ_OK) { lz_segments_destroy(g); return rc; }
    *out = g;
    return LZ_OK;
}

int lz_segments_destroy(lz_segments *g)
{
    if (!g) return LZ_OK;
    cudaFree(g->child_visits); cudaFree(g->root_values); cudaFree(g->len); cudaFree(g->improved_policy);
    delete g;
    return LZ_OK;
}

int lz_segments_store_search_stats(lz_segments *g, const int32_t *d_visits, const float *d_values, const uint8_t *d_active, lz_stream s)
{
    LZ_REQUIRE(g && d_visits && d_values, LZ_EINVAL, "lz_segments_store_search_stats: null argument");
    k_segments_store<<<ceil_div(g->B, 4), 128, 0, (cudaStream_t)s>>>(d_visits, d_values, d_active, g->child_visits, g->root_values, g->len,
                                                                    g->B, g->T, g->A);
    LZ_KERNEL_CHECK();
    return LZ_OK;
}

int lz_segments_reset(lz_segments *g, const uint8_t *d_done, lz_stream s)
{
    LZ_REQUIRE(g, LZ_EINVAL, "lz_segments_reset: null argument");
    k_segments_reset<<<ceil_div(g->B, 256), 256, 0, (cudaStream_t)s>>>(g->len, d_done, g->B);
    LZ_KERNEL_CHECK();
    if (g->improved_policy) {
        const size_t n = (size_t)g->B * g->T * g->A;
        const int blocks = (int)std::min<size_t>((n + 255) / 256, (size_t)kNumSMs * 8);
        k_segments_clear_rows<<<blocks, 256, 0, (cudaStream_t)s>>>(g->improved_policy, d_done, g->B, (size_t)g->T * g->A);
        LZ_KERNEL_CHECK();
    }
    return LZ_OK;
}

int lz_segments_store_improved_policy(lz_segments *g, const float *d_improved_policy, const uint8_t *d_active, lz_stream s)
{
    LZ_REQUIRE(g && d_improved_policy, LZ_EINVAL, "lz_segments_store_improved_policy: null argument");
    if (!g->improved_policy) {
        const size_t n = (size_t)g->B * g->T * g->A;
        int rc = dev_alloc(&g->improved_policy, n);
        if (rc != LZ_OK) return rc;
        LZ_CUDA_CHECK(cudaMemsetAsync(g->improved_policy, 0, n * sizeof(float), (cudaStream_t)s));
    }
    k_segments_store_policy<<<ceil_div(g->B, 4), 128, 0, (cudaStream_t)s>>>(d_improved_policy, d_active, g->improved_policy, g->len,
                                                                           g->B, g->T, g->A);
    LZ_KERNEL_CHECK();
    return LZ_OK;
}

int lz_segments_data(lz_segments *g, float **d_child_visits, float **d_root_values, int32_t **d_len)
{
    LZ_REQUIRE(g, LZ_EINVAL, "lz_segments_data: null argument");
    if (d_child_visits) *d_child_visits = g->child_visits;
    if (d_root_values) *d_root_values = g->root_values;
    if (d_len) *d_len = g->len;
    return LZ_OK;
}

int lz_segments_improved_policy(lz_segments *g, float **d_improved_policy)
{
    LZ_REQUIRE(g && d_improved_policy, LZ_EINVAL, "lz_segments_improved_policy: null argument");
    *d_improved_policy = g->improved_policy;
    return LZ_OK;
}

}  // extern "C"
