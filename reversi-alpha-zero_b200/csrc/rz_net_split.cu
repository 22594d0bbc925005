// rz_net_split.cu -- latency tower for small batches (sm_90a): the function of net_tower_kernel (rz_net_tc.cu), bit for bit,
// with every 2-board tile (M = 128 rows) spread over a cluster of 8 CTAs instead of one CTA.
//
// A single-game search evaluates at most parallel_search_num leaves per wave, i.e. a handful of tiles; the throughput kernel
// then runs one CTA per tile through all convolutions while the other SMs idle.  Here CTA r of a cluster owns output
// channels 32r .. 32r + 31 of every convolution:
//   * weights: the CTA's slice of each packed 32 KB stage of tc_w (8 contiguous 512 B chunks, one per kc: exactly the
//     [kc][n32][j8] B-operand layout) is streamed with cp.async.bulk through a kStages-deep mbarrier ring;
//   * activations: every CTA holds the whole fp16 operand buffer of its tile in the layout (and with the zero border) of
//     net_tower_kernel; two math warpgroups issue wgmma.m64n32k16 over the same K order (tap, kb, j) as the m64n256k16 of
//     the throughput kernel, so each output element sees the same operands and the same fp32 accumulation;
//   * exchange: after a layer's MMAs a cluster barrier marks the operand buffers free; each CTA's epilogue (the same BN,
//     skip and ReLU arithmetic) writes its 32-channel slice of the next operand into all 8 CTAs (st.shared::cluster); a
//     second cluster barrier publishes it.  One operand buffer: two would not fit beside the weight ring;
//   * residual stream: each thread keeps its 2 rows x 8 columns fp32 slice in registers (no global scratch);
//   * head features: the fp32 tower output of the tile is gathered into CTA 0 (over the then idle operand buffer and weight
//     ring), whose threads repeat the head sums of net_tower_kernel in its order (per lane over i = 0..31, then the lane
//     quad) and store the same head features; the dense heads run afterwards in the batched head pass (rz_net_heads.cu).
// Host side: launch_tower_split, one 8-CTA cluster (__cluster_dims__) per tile of the batch capacity, called by the tower
// sequence in rz_net.cu (RZ_NET_IMPL_SPLIT).
#include "rz_bitboard.cuh"
#include "rz_net.cuh"
#include "rz_tc_common.cuh"

namespace rz {
namespace split {
using namespace tc;

constexpr int kCluster = 8;
constexpr int kThreads = 256;
constexpr uint32_t kActCg = 2896, kActSlot = 144;
constexpr uint32_t kActBytes = 32 * kActCg;   // 92,672
constexpr uint32_t kSliceBytes = 4096;        // one stage, 32 output channels
constexpr uint32_t kStages = 12;
constexpr uint32_t kA0Bytes = 8192, kW0Bytes = 2048;
constexpr uint32_t kGatherBytes = 128 * 256 * 4;   // fp32 tower output of the tile (CTA 0, heads)
constexpr uint32_t kOffAct = 0;
constexpr uint32_t kOffW = kOffAct + kActBytes;
constexpr uint32_t kOffA0 = kOffW + kStages * kSliceBytes;
constexpr uint32_t kOffW0 = kOffA0 + kA0Bytes;
constexpr uint32_t kOffBar = kOffW0 + kW0Bytes;
constexpr uint32_t kNumBars = 2 * kStages + 1;           // full[], empty[], w0
constexpr uint32_t kSmemBytes = kOffBar + kNumBars * 8;
constexpr uint32_t kSmemAlloc = kSmemBytes + 128;
static_assert(kOffW + kStages * kSliceBytes >= kGatherBytes, "gather buffer must fit over the operand buffer and the ring");
static_assert(kSmemAlloc <= 232448, "shared memory budget exceeded");

__device__ __forceinline__ void wgmma_m64n32k16(float (&d)[16], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %18, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 {"
        "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1, 0, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]),
          "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
        : "l"(adesc), "l"(bdesc), "r"(accumulate)
        : "memory");
}
__device__ __forceinline__ void acc_fence16(float (&d)[16]) {
#pragma unroll
    for (int i = 0; i < 16; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
__device__ __forceinline__ uint32_t mapa(uint32_t addr, uint32_t rank) {
    uint32_t r;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(addr), "r"(rank));
    return r;
}
__device__ __forceinline__ void st_cluster_b32(uint32_t addr, uint32_t v) {
    asm volatile("st.shared::cluster.b32 [%0], %1;" ::"r"(addr), "r"(v) : "memory");
}
__device__ __forceinline__ void st_cluster_v2f(uint32_t addr, float a, float b) {
    asm volatile("st.shared::cluster.v2.f32 [%0], {%1, %2};" ::"r"(addr), "f"(a), "f"(b) : "memory");
}

// grid = kCluster CTAs per tile of the batch capacity; a cluster whose tile starts past the (device-side) count leaves at once
__global__ void __cluster_dims__(kCluster, 1, 1) __launch_bounds__(kThreads, 1) net_split_kernel(const Params pp) {
    Params p = pp;
    if (p.n_dev) p.n = *p.n_dev;
    const uint32_t tile = blockIdx.x / kCluster;
    const uint32_t pos0 = tile * 2;
    if (pos0 >= p.n) return;   // the whole cluster: no barrier or remote access has happened yet
    extern __shared__ uint8_t smem_raw[];
    const uint32_t base = (smem_u32(smem_raw) + 127u) & ~127u;
    uint8_t* sm = smem_raw + (base - smem_u32(smem_raw));
    const uint32_t crank = cluster_ctarank();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, et = threadIdx.x;
    const uint32_t bar0 = base + kOffBar;
    auto bar_full = [&](uint32_t s) { return bar0 + s * 8; };
    auto bar_empty = [&](uint32_t s) { return bar0 + (kStages + s) * 8; };
    const uint32_t bar_w0 = bar0 + 2 * kStages * 8;
    const int L = p.n_layers;
    const uint32_t total = (uint32_t)(L - 1) * 36;   // weight stages of the tower
    const uint8_t* wsrc = reinterpret_cast<const uint8_t*>(p.w) + crank * 512;

    auto issue = [&](uint32_t t) {   // stage t of the tower, this CTA's 32 output channels
        const uint32_t slot = t % kStages;
        const uint8_t* src = wsrc + (size_t)t * 32768;
        mbar_expect_tx(bar_full(slot), kSliceBytes);
#pragma unroll
        for (uint32_t kc = 0; kc < 8; ++kc) bulk_g2s(base + kOffW + slot * kSliceBytes + kc * 512, src + kc * 4096, 512, bar_full(slot));
    };

    for (uint32_t i = threadIdx.x * 16; i < kActBytes; i += kThreads * 16) *reinterpret_cast<uint4*>(sm + kOffAct + i) = make_uint4(0, 0, 0, 0);
    if (threadIdx.x == 0) {
        for (uint32_t s = 0; s < kStages; ++s) { mbar_init(bar_full(s), 1); mbar_init(bar_empty(s), 8); }
        mbar_init(bar_w0, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        mbar_expect_tx(bar_w0, kW0Bytes);
        const uint8_t* w0 = reinterpret_cast<const uint8_t*>(p.w0) + crank * 512;
        for (uint32_t kc = 0; kc < 4; ++kc) bulk_g2s(base + kOffW0 + kc * 512, w0 + kc * 4096, 512, bar_w0);
        for (uint32_t t = 0; t < kStages && t < total; ++t) issue(t);
    }
    {   // layer-0 operand: the same im2col tile as net_tower_kernel
        const int m = et & 127, g = m >> 3, brd = g & 1;
        const bool valid = pos0 + brd < p.n;
        build_layer0_operand(sm + kOffA0, valid ? p.own[pos0 + brd] : 0, valid ? p.enemy[pos0 + brd] : 0, 2 * (et >> 7), g, m & 7, g >> 1);
    }
    fence_proxy_async();
    cluster_sync_all();   // every CTA's operand buffer is zeroed before any peer writes into it

    const int wg = warp >> 2;
    const int r0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);
    const int g0 = r0 >> 3, x = r0 & 7, y = g0 >> 1;
    const int cq = 2 * (lane & 3);
    const uint32_t act_row0 = base + kOffAct + (g0 + 2) * kActSlot + (x + 1) * 16 + cq * 2;   // + cg * kActCg
    const uint32_t act_row1 = act_row0 + kActSlot;
    const uint32_t a_wg = base + kOffAct + wg * 8 * kActSlot;
    float d[16], res[16];
    uint32_t t = 0;   // weight stage being consumed
    for (int l = 0; l < L; ++l) {
        acc_fence16(d);
        if (l == 0) {
            mbar_wait(bar_w0, 0);
            wgmma_fence();
#pragma unroll
            for (uint32_t j = 0; j < 2; ++j)
                wgmma_m64n32k16(d, smem_desc(base + kOffA0 + j * 2 * 2048 + wg * 1024, 2048, 128), smem_desc(base + kOffW0 + j * 2 * 512, 512, 128), j);
            wgmma_commit();
            wgmma_wait<0>();
        } else {
            for (uint32_t tap = 0; tap < 9; ++tap) {
                const uint32_t a_tap = a_wg + (2 * (tap / 3)) * kActSlot + (tap % 3) * 16;
                for (uint32_t kb = 0; kb < 4; ++kb, ++t) {
                    const uint32_t slot = t % kStages;
                    mbar_wait(bar_full(slot), (t / kStages) & 1);
                    const uint32_t b_st = base + kOffW + slot * kSliceBytes;
                    wgmma_fence();
#pragma unroll
                    for (uint32_t j = 0; j < 4; ++j)
                        wgmma_m64n32k16(d, smem_desc(a_tap + (kb * 8 + 2 * j) * kActCg, kActCg, kActSlot), smem_desc(b_st + 2 * j * 512, 512, 128),
                                        (tap | kb | j) != 0);
                    wgmma_commit();
                    wgmma_wait<1>();   // stage t - 1's MMAs are done: its slot may be refilled with stage t - 1 + kStages
                    if (t > 0) {
                        const uint32_t pt = t - 1;
                        if (lane == 0) mbar_arrive(bar_empty(pt % kStages));
                        if (threadIdx.x == 0 && pt + kStages < total) {
                            mbar_wait(bar_empty(pt % kStages), (pt / kStages) & 1);
                            issue(pt + kStages);
                        }
                        __syncwarp();
                    }
                }
            }
            wgmma_wait<0>();
        }
        acc_fence16(d);
        cluster_sync_all();   // every CTA has finished reading its operand buffer (and, after the last layer, its ring)
        const bool is_conv2 = l > 0 && (l & 1) == 0;
        const bool keep_res = l == 0 || is_conv2;
        const bool last = l == L - 1;
        const float* sc = p.ss + (size_t)l * 512;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int c = (int)crank * 32 + 8 * i + cq;
            const float2 s = __ldg(reinterpret_cast<const float2*>(sc + c));
            const float2 b = __ldg(reinterpret_cast<const float2*>(sc + 256 + c));
            float v0 = fmaf(d[4 * i + 0], s.x, b.x), v1 = fmaf(d[4 * i + 1], s.y, b.y);
            float v2 = fmaf(d[4 * i + 2], s.x, b.x), v3 = fmaf(d[4 * i + 3], s.y, b.y);
            if (is_conv2) {
                v0 += res[4 * i + 0]; v1 += res[4 * i + 1]; v2 += res[4 * i + 2]; v3 += res[4 * i + 3];
            }
            if (keep_res || last) {
                v0 = fmaxf(v0, 0.f); v1 = fmaxf(v1, 0.f); v2 = fmaxf(v2, 0.f); v3 = fmaxf(v3, 0.f);
            }
            if (!last) {
                if (keep_res) { res[4 * i + 0] = v0; res[4 * i + 1] = v1; res[4 * i + 2] = v2; res[4 * i + 3] = v3; }
                const uint32_t h0 = keep_res ? pack_h2<false>(v0, v1) : pack_h2<true>(v0, v1);
                const uint32_t h1 = keep_res ? pack_h2<false>(v2, v3) : pack_h2<true>(v2, v3);
                const uint32_t off = (uint32_t)(c >> 3) * kActCg;
#pragma unroll
                for (uint32_t q = 0; q < kCluster; ++q) {
                    st_cluster_b32(mapa(act_row0 + off, q), h0);
                    st_cluster_b32(mapa(act_row1 + off, q), h1);
                }
            } else {   // fp32 tower output -> CTA 0, [row][256 channels]
                st_cluster_v2f(mapa(base + ((uint32_t)r0 * 256 + c) * 4, 0), v0, v1);
                st_cluster_v2f(mapa(base + ((uint32_t)(r0 + 8) * 256 + c) * 4, 0), v2, v3);
            }
        }
        asm volatile("fence.proxy.async;" ::: "memory");
        cluster_sync_all();   // the next operand (or the gathered tower output) is complete in every CTA
        fence_proxy_async();
    }
    if (crank != 0) return;   // no peer touches this CTA any more

    // ---- head features on CTA 0, in the summation order of net_tower_kernel ---------------------------
    const float* gat = reinterpret_cast<const float*>(sm);
    const float* pw = p.blob + p.off_policy_conv;
    const float* vw = p.blob + p.off_value_conv;
    float hs[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    float* dbg0 = nullptr;
    float* dbg1 = nullptr;
    if (p.dbg_tower) {
        if (pos0 < p.n) dbg0 = p.dbg_tower + ((size_t)pos0 * 64 + y * 8 + x) * 256;
        if (pos0 + 1 < p.n) dbg1 = p.dbg_tower + ((size_t)(pos0 + 1) * 64 + y * 8 + x) * 256;
    }
#pragma unroll 4
    for (int i = 0; i < 32; ++i) {
        const int c = 8 * i + cq;
        const float2 a = *reinterpret_cast<const float2*>(gat + r0 * 256 + c);
        const float2 b = *reinterpret_cast<const float2*>(gat + (r0 + 8) * 256 + c);
        const float v0 = a.x, v1 = a.y, v2 = b.x, v3 = b.y;
        const float4 w = __ldg(reinterpret_cast<const float4*>(pw + 2 * c));
        const float2 wv = make_float2(__ldg(vw + c), __ldg(vw + c + 1));
        hs[0] = fmaf(v1, w.z, fmaf(v0, w.x, hs[0]));
        hs[1] = fmaf(v1, w.w, fmaf(v0, w.y, hs[1]));
        hs[2] = fmaf(v1, wv.y, fmaf(v0, wv.x, hs[2]));
        hs[3] = fmaf(v3, w.z, fmaf(v2, w.x, hs[3]));
        hs[4] = fmaf(v3, w.w, fmaf(v2, w.y, hs[4]));
        hs[5] = fmaf(v3, wv.y, fmaf(v2, wv.x, hs[5]));
        if (dbg0) *reinterpret_cast<float2*>(dbg0 + c) = make_float2(v0, v1);
        if (dbg1) *reinterpret_cast<float2*>(dbg1 + c) = make_float2(v2, v3);
    }
#pragma unroll
    for (int k = 0; k < 6; ++k) {
        hs[k] += __shfl_xor_sync(0xffffffffu, hs[k], 1);
        hs[k] += __shfl_xor_sync(0xffffffffu, hs[k], 2);
    }
    const int q = lane & 3;
    if (q < 2 && pos0 + q < p.n)   // + 0.f as in net_tower_kernel
        store_head_features(p.feat + (size_t)(pos0 + q) * kHeadFeatures, p.ss + (size_t)L * 512, y * 8 + x, hs[3 * q] + 0.f,
                            hs[3 * q + 1] + 0.f, hs[3 * q + 2] + 0.f);
}

}  // namespace split

int tc::launch_tower_split(const Params& p, cudaStream_t stream) {
    static bool attr = false;
    if (!attr) {
        RZ_CUDA_TRY(cudaFuncSetAttribute(split::net_split_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)split::kSmemAlloc));
        attr = true;
    }
    const uint32_t ntiles = (p.n + 1) / 2;
    split::net_split_kernel<<<ntiles * split::kCluster, split::kThreads, split::kSmemAlloc, stream>>>(p);
    RZ_LAUNCH_CHECK();
    return RZ_OK;
}

}  // namespace rz
