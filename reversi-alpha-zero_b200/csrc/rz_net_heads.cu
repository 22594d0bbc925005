// rz_net_heads.cu -- the dense heads of the wgmma towers (rz_net_tc.cu, rz_net_tc_narrow.cu, rz_net_split.cu) as one
// batched pass over the head features the tower stored (agent/model.py:48-56): Dense(128 -> 64) + softmax for the policy,
// Dense(64 -> V) + ReLU -> Dense(V -> 1) + tanh for the value.
//
// Run inside a tower tile, these layers read ~96 KB of Dense weights from L2 for two boards and ran on dependent fmaf
// chains behind CTA barriers while the tensor cores idled.  Here a CTA stages the weights in shared memory once and a
// warp carries kBoards boards at a time, so every weight read from shared memory feeds kBoards FMAs (2 kBoards for the
// policy).  Every output is the same sequence of fp32 operations as in the tower: each sum runs over its inputs in index
// order from the bias (the fc2 partials from 0), the softmax and the fc2 reduction use the same xor trees, and this file
// is compiled with the towers' flags (not -fmad=false), so the outputs are bit-identical to the per-tile heads.
#include "rz_net.cuh"
#include "rz_tc_common.cuh"

namespace rz {
namespace heads {

constexpr int kThreads = 512;
constexpr int kWarps = kThreads / 32;
constexpr int kBoards = 4;   // boards per warp task
// shared memory, in floats: policy kernel [128][64], policy bias [64], value fc1 kernel [64][V], fc1 bias [V], fc2 kernel [V],
// then per warp its task's head features transposed to [192][kBoards] (a float4 load gives one feature of all kBoards boards)
constexpr uint32_t kOffPb = 128 * 64;
constexpr uint32_t kOffK1 = kOffPb + 64;
__host__ __device__ constexpr uint32_t off_feat(int V) { return (kOffK1 + 66u * (uint32_t)V + 3u) & ~3u; }
__host__ __device__ constexpr uint32_t smem_bytes(int V) { return (off_feat(V) + kWarps * kHeadFeatures * kBoards) * 4u; }
static_assert(smem_bytes(tc::kTcMaxV) <= 232448, "shared memory budget exceeded");

__device__ __forceinline__ void stage(float* dst, const float* src, int count) {
#pragma unroll 4
    for (int i = threadIdx.x; i < count; i += kThreads) dst[i] = __ldg(src + i);
}

__global__ void __launch_bounds__(kThreads, 1) heads_kernel(const tc::Params p) {
    const uint32_t n = p.n_dev ? *p.n_dev : p.n;
    const int V = p.V;
    extern __shared__ float4 smem4[];
    float* sm = reinterpret_cast<float*>(smem4);
    const float* kp = sm;
    const float* bp = sm + kOffPb;
    const float* k1 = sm + kOffK1;
    const float* b1 = k1 + 64 * V;
    const float* k2 = b1 + V;
    stage(sm, p.blob + p.off_policy_fc_k, 128 * 64);
    stage(sm + kOffPb, p.blob + p.off_policy_fc_b, 64);
    stage(sm + kOffK1, p.blob + p.off_value_fc1_k, 64 * V);
    stage(sm + kOffK1 + 64 * V, p.blob + p.off_value_fc1_b, V);
    stage(sm + kOffK1 + 65 * V, p.blob + p.off_value_fc2_k, V);
    __syncthreads();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    float* ft = sm + off_feat(V) + warp * kHeadFeatures * kBoards;
    const float b2 = __ldg(p.blob + p.off_value_fc2_b);

    for (uint32_t b0 = (blockIdx.x * kWarps + warp) * kBoards; b0 < n; b0 += gridDim.x * kWarps * kBoards) {
        __syncwarp();   // the previous task's reads of ft are done
        for (int k = lane; k < kHeadFeatures * kBoards; k += 32) {
            const int b = k / kHeadFeatures, i = k - b * kHeadFeatures;
            ft[i * kBoards + b] = b0 + b < n ? p.feat[(size_t)(b0 + b) * kHeadFeatures + i] : 0.f;
        }
        __syncwarp();
        // policy logits: lane l holds logits l and l + 32 of every board, the softmax's lane assignment
        float lg[kBoards][2];
#pragma unroll
        for (int b = 0; b < kBoards; ++b) { lg[b][0] = bp[lane]; lg[b][1] = bp[32 + lane]; }
#pragma unroll 8
        for (int i = 0; i < 128; ++i) {
            const float4 h = *reinterpret_cast<const float4*>(ft + i * kBoards);
            const float w0 = kp[i * 64 + lane], w1 = kp[i * 64 + 32 + lane];
            const float hb[kBoards] = {h.x, h.y, h.z, h.w};
#pragma unroll
            for (int b = 0; b < kBoards; ++b) {
                lg[b][0] = fmaf(hb[b], w0, lg[b][0]);
                lg[b][1] = fmaf(hb[b], w1, lg[b][1]);
            }
        }
#pragma unroll
        for (int b = 0; b < kBoards; ++b) {   // softmax over 64 logits
            const float l0 = lg[b][0], l1 = lg[b][1];
            float mx = fmaxf(l0, l1);
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
            const float e0 = expf(l0 - mx), e1 = expf(l1 - mx);
            float s = e0 + e1;
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
            if (b0 + b < n) {
                p.policy[(size_t)(b0 + b) * 64 + lane] = e0 / s;
                p.policy[(size_t)(b0 + b) * 64 + 32 + lane] = e1 / s;
                if (p.dbg_logits) {
                    p.dbg_logits[(size_t)(b0 + b) * 64 + lane] = l0;
                    p.dbg_logits[(size_t)(b0 + b) * 64 + 32 + lane] = l1;
                }
            }
        }
        // value: lane l computes fc1 outputs j = l, l + 32, ... and folds each into its fc2 partial in that order
        float acc[kBoards];
#pragma unroll
        for (int b = 0; b < kBoards; ++b) acc[b] = 0.f;
        for (int j = lane; j < V; j += 32) {
            float f[kBoards];
#pragma unroll
            for (int b = 0; b < kBoards; ++b) f[b] = b1[j];
#pragma unroll 8
            for (int i = 0; i < 64; ++i) {
                const float4 h = *reinterpret_cast<const float4*>(ft + (128 + i) * kBoards);
                const float w = k1[i * V + j];
                const float hb[kBoards] = {h.x, h.y, h.z, h.w};
#pragma unroll
                for (int b = 0; b < kBoards; ++b) f[b] = fmaf(hb[b], w, f[b]);
            }
            const float w2 = k2[j];
#pragma unroll
            for (int b = 0; b < kBoards; ++b) acc[b] = fmaf(fmaxf(f[b], 0.f), w2, acc[b]);
        }
#pragma unroll
        for (int b = 0; b < kBoards; ++b) {
            float a = acc[b];
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
            if (lane == 0 && b0 + b < n) {
                const float pre = a + b2;
                p.value[b0 + b] = tanhf(pre);
                if (p.dbg_vlogit) p.dbg_vlogit[b0 + b] = pre;
            }
        }
    }
}
static_assert(kBoards == 4, "the feature tile is read as one float4 per feature");

}  // namespace heads

int net_heads(const tc::Params& p, cudaStream_t stream) {
    static bool attr = false;
    if (!attr) {
        RZ_CUDA_TRY(cudaFuncSetAttribute(heads::heads_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)heads::smem_bytes(tc::kTcMaxV)));
        attr = true;
    }
    constexpr uint32_t kPerCta = heads::kWarps * heads::kBoards;
    const uint32_t ctas = (p.n + kPerCta - 1) / kPerCta;
    if (ctas == 0) return RZ_OK;
    heads::heads_kernel<<<ctas < (uint32_t)num_sms() ? ctas : (uint32_t)num_sms(), heads::kThreads, heads::smem_bytes(p.V), stream>>>(p);
    RZ_LAUNCH_CHECK();
    return RZ_OK;
}

}  // namespace rz
