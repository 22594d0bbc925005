// rz_net_tc_narrow.cu -- the fused persistent wgmma tower of rz_net_tc.cu for the 64- and 128-filter networks (sm_90a).
//
// Same machine as net_tower_kernel (rz_net_tc.cu; DESIGN.md §5), with the tile widened so that every MMA keeps the
// 128-row x 256-column accumulator footprint of the 256-filter kernel:
//   * a tile holds B = 512 / F boards (4 at 128 filters, 8 at 64): M = 64 B pixel rows, two math warpgroups of 32 B rows;
//   * each math warpgroup issues T = 256 / F wgmma.m64nFk16 per k-step, one per 64-row sub-tile, all with the same B
//     (weight) descriptor; sub-tile t accumulates into d[t * F/2 ...] of the thread's 128 fp32 registers;
//   * activations: fp16, K-major no-swizzle, one-pixel zero border, slot = B*(y+1) + board (a dy shift is B slots):
//         chunk(cg, slot, xp) at cg*kActCg + slot*144 + xp*16,  kActCg = B*10*144 + 16  (92.4 KB / 92.3 KB)
//     MMA row m = (B*y + board)*8 + x; rows r and r + 8 of a thread are the same pixel of boards b and b + 1 (b even);
//   * weights: fp16 stages of TPS taps x F input x F output channels streamed through a 3-deep mbarrier ring by one
//     producer thread (multicast across a CTA pair with CL = 2): one tap (32 KB, 9 stages per conv) at 128 filters, one
//     kernel row of three taps (24 KB, 3 stages per conv) at 64 filters;
//   * epilogue (folded BN, skip connection from the per-CTA fp32 residual scratch, ReLU, fp16 operand for the next layer),
//     layer 0 (im2col GEMM, K = 18 padded to 32) and head features as in rz_net_tc.cu, for B boards.  A row's 1x1
//     head-conv sums are complete in its lane quad, so they need no cross-warpgroup partial-sum array.  The dense heads
//     run afterwards as one batched pass (rz_net_heads.cu).
// Every output element goes through the same operations whichever tile slot its board lands in.
// Host side: launch_tower_narrow, the CTA-pair launch of rz_net_tc.cu (launch_tower_pairs, rz_tc_common.cuh) with B-board
// tiles, called by the tower sequence in rz_net.cu.  rz_net.cu also packs the weights at load, in the one layout of every
// width (tc_w, rz_net.cuh).
#include <type_traits>
#include "rz_bitboard.cuh"
#include "rz_net.cuh"
#include "rz_tc_common.cuh"

namespace rz {
namespace tc {
namespace narrow {

constexpr uint32_t kProducerRegs = 40, kMathRegs = 232;
constexpr uint32_t kActSlot = 144;
constexpr uint32_t kStages = 3;
constexpr int kResAhead = 4;

template <int F>
struct Cfg {
    static_assert(F == 64 || F == 128, "narrow tower: 64 or 128 filters");
    static constexpr int B = 512 / F;                 // boards per tile
    static constexpr int T = 256 / F;                 // 64-row sub-tiles (MMAs per k-step) per math warpgroup
    static constexpr int TPS = F == 128 ? 1 : 3;      // taps per weight stage
    static constexpr int S = 9 / TPS;                 // weight stages per conv layer
    static constexpr int KPT = F / 16;                // k16 steps per tap
    static constexpr uint32_t kActCg = B * 10 * kActSlot + 16;
    static constexpr uint32_t kActBytes = (F / 8) * kActCg;
    static constexpr uint32_t kTapBytes = F * F * 2;  // one tap's [F/8 kc][F n][8] fp16 image
    static constexpr uint32_t kStageBytes = TPS * kTapBytes;
    static constexpr uint32_t kA0Kc = B * 8 * 128;    // layer-0 operand: bytes per 8-wide K chunk (8B board rows x 8 x 16 B)
    static constexpr uint32_t kA0Bytes = 4 * kA0Kc;
    static constexpr uint32_t kW0Bytes = 4 * F * 16;
    static constexpr uint32_t kOffAct = 0;
    static constexpr uint32_t kOffW = kOffAct + kActBytes;
    static constexpr uint32_t kOffA0 = kOffW + kStages * kStageBytes;
    static constexpr uint32_t kOffW0 = kOffA0 + kA0Bytes;
    static constexpr uint32_t kOffSS = kOffW0 + kW0Bytes;           // 2 x [scale F][shift F] fp32
    static constexpr uint32_t kOffHw = kOffSS + 2 * 2 * F * 4;      // 1x1 head-conv weights: policy [F][2], value [F] fp32
    static constexpr uint32_t kOffFeat = kOffHw + 3 * F * 4;        // [B][kHeadFeatures] head features of the tile
    static constexpr uint32_t kOffBar = kOffFeat + B * kHeadFeatures * 4;   // full[], empty[], w0
    static constexpr uint32_t kSmemBytes = kOffBar + (2 * kStages + 1) * 8;
    static constexpr uint32_t kSmemAlloc = kSmemBytes + 128;        // slack for manual 128 B alignment
    static_assert(kSmemAlloc <= 232448, "shared memory budget exceeded");
    static_assert(kActBytes % 16 == 0 && kOffW % 128 == 0 && kStageBytes % (16 * 2) == 0 && kOffA0 % 128 == 0 && kOffW0 % 128 == 0,
                  "operand and bulk-copy alignment");
    static_assert(T * F / 2 == 128 && T * (F / 8) == 32, "128 accumulators = 32 residual float4 per thread");
};
static_assert(kTowerResFloatsPerCta == (size_t)256 * 128, "residual scratch per CTA");

// the 256 / F MMAs of one k-step of a math warpgroup: sub-tile t reads the A rows at a + t * a_step and accumulates into
// d[t * F/2 ..]; all of them share the weight descriptor
template <int F>
__device__ __forceinline__ void mma_kstep(float (&d)[128], uint32_t a, uint32_t a_step, uint32_t lbo, uint32_t sbo, uint64_t bdesc,
                                          uint32_t accumulate) {
    if constexpr (F == 128) {
        wgmma_m64n128k16<0>(d, smem_desc(a, lbo, sbo), bdesc, accumulate);
        wgmma_m64n128k16<64>(d, smem_desc(a + a_step, lbo, sbo), bdesc, accumulate);
    } else {
        wgmma_m64n64k16<0>(d, smem_desc(a, lbo, sbo), bdesc, accumulate);
        wgmma_m64n64k16<32>(d, smem_desc(a + a_step, lbo, sbo), bdesc, accumulate);
        wgmma_m64n64k16<64>(d, smem_desc(a + 2 * a_step, lbo, sbo), bdesc, accumulate);
        wgmma_m64n64k16<96>(d, smem_desc(a + 3 * a_step, lbo, sbo), bdesc, accumulate);
    }
}

// layer-0 im2col of one board row (g, x) for K chunks kc0, kc0 + 1 (build_layer0_operand with a K-chunk stride of kKc)
template <uint32_t kKc>
__device__ __forceinline__ void build_layer0_rows(uint8_t* a0, u64 o, u64 e, int kc0, int g, int x, int y) {
#pragma unroll
    for (int kk = 0; kk < 2; ++kk) {
        const int kc = kc0 + kk;
        uint32_t w[4];
#pragma unroll
        for (int jp = 0; jp < 4; ++jp) {
            uint32_t packed = 0;
#pragma unroll
            for (int half = 0; half < 2; ++half) {
                const int k = kc * 8 + jp * 2 + half;
                uint32_t bit = 0;
                if (k < 18) {
                    const int tap = k >> 1, yy = y + tap / 3 - 1, xx = x + tap % 3 - 1;
                    if (yy >= 0 && yy < 8 && xx >= 0 && xx < 8) bit = (uint32_t)((((k & 1) ? e : o) >> (yy * 8 + xx)) & 1ULL);
                }
                packed |= (bit ? 0x3C00u : 0u) << (16 * half);  // fp16 1.0
            }
            w[jp] = packed;
        }
        *reinterpret_cast<uint4*>(a0 + kc * kKc + g * 128 + x * 16) = make_uint4(w[0], w[1], w[2], w[3]);
    }
}

// CL = thread-block-cluster size (1 or 2), as in net_tower_kernel
template <int F, int CL>
__global__ void __launch_bounds__(kThreads, 1) net_tower_narrow_kernel(const Params pp) {
    using C = Cfg<F>;
    constexpr int B = C::B, T = C::T;
    Params p = pp;
    if (p.n_dev) p.n = *p.n_dev;
    extern __shared__ uint8_t smem_raw[];
    const uint32_t base = (smem_u32(smem_raw) + 127u) & ~127u;
    uint8_t* sm = smem_raw + (base - smem_u32(smem_raw));
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t bar0 = base + C::kOffBar;
    auto bar_full = [&](uint32_t s) { return bar0 + s * 8; };
    auto bar_empty = [&](uint32_t s) { return bar0 + (kStages + s) * 8; };
    const uint32_t bar_w0 = bar0 + 2 * kStages * 8;
    const uint32_t ntiles = (p.n + B - 1) / B;
    const int L = p.n_layers;
    const uint32_t crank = CL > 1 ? cluster_ctarank() : 0u;
    const uint32_t cbase = blockIdx.x - crank;
    const uint32_t iters = cbase < ntiles ? (ntiles - cbase + gridDim.x - 1) / gridDim.x : 0u;

    // ---- one-time setup -----------------------------------------------------------------------------
    for (uint32_t i = threadIdx.x * 16; i < C::kActBytes; i += kThreads * 16) *reinterpret_cast<uint4*>(sm + C::kOffAct + i) = make_uint4(0, 0, 0, 0);
    fence_proxy_async();
    for (uint32_t i = threadIdx.x; i < 3 * F; i += kThreads)
        reinterpret_cast<float*>(sm + C::kOffHw)[i] = __ldg(i < 2 * F ? p.blob + p.off_policy_conv + i : p.blob + p.off_value_conv + (i - 2 * F));
    if (threadIdx.x == 0) {
        for (uint32_t s = 0; s < kStages; ++s) { mbar_init(bar_full(s), 1); mbar_init(bar_empty(s), 8 * CL); }
        mbar_init(bar_w0, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    if (CL > 1) cluster_sync_all();

    if (warp >= 8) {
        // ===== weight producer =====================================================================
        asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(kProducerRegs));
        if (warp == 8 && lane == 0) {
            if (iters > 0) {
                mbar_expect_tx(bar_w0, C::kW0Bytes);
                bulk_g2s(base + C::kOffW0, p.w0, C::kW0Bytes, bar_w0);
            }
            uint32_t stage = 0, phase = 0;
            for (uint32_t it = 0; it < iters; ++it) {
                for (int l = 1; l < L; ++l) {
                    const uint8_t* src = reinterpret_cast<const uint8_t*>(p.w) + (size_t)(l - 1) * C::S * C::kStageBytes;
                    for (int s = 0; s < C::S; ++s) {
                        mbar_wait(bar_empty(stage), phase ^ 1);
                        mbar_expect_tx(bar_full(stage), C::kStageBytes);
                        if (CL == 1) {
                            bulk_g2s(base + C::kOffW + stage * C::kStageBytes, src + (size_t)s * C::kStageBytes, C::kStageBytes, bar_full(stage));
                        } else {
                            constexpr uint32_t kSlice = C::kStageBytes / CL;
                            bulk_g2s_mc(base + C::kOffW + stage * C::kStageBytes + crank * kSlice, src + (size_t)s * C::kStageBytes + crank * kSlice,
                                        kSlice, bar_full(stage), (uint16_t)((1u << CL) - 1u));
                        }
                        if (++stage == kStages) { stage = 0; phase ^= 1; }
                    }
                }
            }
        }
    } else {
        // ===== math warpgroups (2) =================================================================
        asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(kMathRegs));
        const int et = threadIdx.x;   // 0..255
        const int wg = warp >> 2;     // MMA rows wg*64T .. wg*64T + 64T - 1
        const int x = lane >> 2, cq = 2 * (lane & 3);
        // sub-tile t: board rows g_t = g0 + 8t (board g_t % B at y = g_t / B) and g_t + 1 (the next board), pixel column x
        const int g0 = wg * T * 8 + (warp & 3) * 2;
        const uint32_t act_row0 = base + C::kOffAct + (g0 + B) * kActSlot + (x + 1) * 16 + cq * 2;  // + 8t*kActSlot + cg*kActCg
        const uint32_t a_wg = base + C::kOffAct + wg * T * 8 * kActSlot;                            // + 8t*kActSlot: sub-tile t
        float* ss_s = reinterpret_cast<float*>(sm + C::kOffSS);
        float4* res = reinterpret_cast<float4*>(p.res + (size_t)blockIdx.x * kTowerResFloatsPerCta) + et;   // + k * 256
        const float* hw = reinterpret_cast<const float*>(sm + C::kOffHw);
        float* feat_s = reinterpret_cast<float*>(sm + C::kOffFeat);
        const float* ssh = p.ss + (size_t)L * 2 * F;   // folded BN of the head convolutions
        uint32_t stage = 0, phase = 0, ss_buf = 0;
        float d[128];
        if (et < 2 * F) ss_s[et] = __ldg(p.ss + et);

        for (uint32_t it = 0; it < iters; ++it) {
            const uint32_t tile = blockIdx.x + it * gridDim.x;
            const uint32_t pos0 = tile * B;
            for (int idx = et; idx < 2 * 64 * B; idx += 256) {   // (row m, K-chunk pair) of the layer-0 im2col tile
                const int m = idx & (64 * B - 1), g = m >> 3, brd = g % B;
                const bool valid = pos0 + brd < p.n;
                build_layer0_rows<C::kA0Kc>(sm + C::kOffA0, valid ? p.own[pos0 + brd] : 0, valid ? p.enemy[pos0 + brd] : 0,
                                            2 * (idx / (64 * B)), g, m & 7, g / B);
            }
            fence_proxy_async();
            for (int l = 0; l < L; ++l) {
                const float* sc = ss_s + ss_buf * 2 * F;
                const bool is_conv2 = l > 0 && (l & 1) == 0;
                float4 rb[kResAhead];
                epi_bar();
                if (et < 2 * F) {
                    const size_t nl = l + 1 < L ? (size_t)l + 1 : 0;
                    cp_async_4(smem_u32(ss_s + (ss_buf ^ 1) * 2 * F + et), p.ss + nl * 2 * F + et);
                }
                acc_fence(d);
                if (l == 0) {
                    mbar_wait(bar_w0, 0);
                    wgmma_fence();
#pragma unroll
                    for (uint32_t j = 0; j < 2; ++j)
                        mma_kstep<F>(d, base + C::kOffA0 + j * 2 * C::kA0Kc + wg * T * 1024, 1024, C::kA0Kc, 128,
                                     smem_desc(base + C::kOffW0 + j * 2 * F * 16, F * 16, 128), j);
                    wgmma_commit();
                    wgmma_wait<0>();
                } else {
                    int prev = -1;
                    for (int s = 0; s < C::S; ++s) {
                        // stage s = taps (kh, kw0 .. kw0 + TPS - 1); tap (kh, kw) reads slot offset B*kh, chunk offset kw
                        const int kh = C::TPS == 3 ? s : s / 3, kw0 = C::TPS == 3 ? 0 : s % 3;
                        const uint32_t a_st = a_wg + B * kh * kActSlot + kw0 * 16;
                        mbar_wait(bar_full(stage), phase);
                        const uint32_t b_st = base + C::kOffW + stage * C::kStageBytes;
                        wgmma_fence();
#pragma unroll
                        for (int ks = 0; ks < C::TPS * C::KPT; ++ks) {
                            const int tt = ks / C::KPT, kk = ks % C::KPT;
                            mma_kstep<F>(d, a_st + tt * 16 + 2 * kk * C::kActCg, 8 * kActSlot, C::kActCg, kActSlot,
                                         smem_desc(b_st + tt * C::kTapBytes + 2 * kk * F * 16, F * 16, 128), (s | ks) != 0);
                        }
                        wgmma_commit();
                        wgmma_wait<1>();
                        if (prev >= 0 && lane == 0) {
                            mbar_arrive(bar_empty(prev));
                            if (CL > 1) mbar_arrive_cta(bar_empty(prev), crank ^ 1u);
                        }
                        prev = (int)stage;
                        if (++stage == kStages) { stage = 0; phase ^= 1; }
                    }
                    if (is_conv2) {
#pragma unroll
                        for (int i = 0; i < kResAhead; ++i) rb[i] = res[i * 256];
                    }
                    wgmma_wait<0>();
                    if (lane == 0) {
                        mbar_arrive(bar_empty(prev));
                        if (CL > 1) mbar_arrive_cta(bar_empty(prev), crank ^ 1u);
                    }
                }
                acc_fence(d);
                cp_async_wait_all();
                ss_buf ^= 1;
                const bool keep_res = l == 0 || is_conv2;
                const bool last = l == L - 1;
                if (!last) epi_bar();
                // compiled once per layer kind (see rz_net_tc.cu); flat step k = t * F/8 + i covers channel 8i + cq of sub-tile t:
                // accumulators d[4k .. 4k + 3], residual float4 k.  The last layer finishes sub-tile t's head 1x1 sums (and
                // stores its head features) as soon as its channels are done, so that only six sums are live at a time.
                constexpr int kEpiRelu = 0, kEpiKeep = 1, kEpiLast = 2;
                auto epilogue = [&](auto conv2, auto kind) {
                    constexpr bool kConv2 = decltype(conv2)::value;
                    constexpr bool kKeep = decltype(kind)::value == kEpiKeep, kLast = decltype(kind)::value == kEpiLast;
                    float hs[6];   // head sums (policy 0, policy 1, value) x (board b_t, b_t + 1) of the current sub-tile
#pragma unroll
                    for (int k = 0; k < 32; ++k) {
                        const int t = k / (F / 8), c = 8 * (k % (F / 8)) + cq;
                        if (kLast && c == cq) {
#pragma unroll
                            for (int h = 0; h < 6; ++h) hs[h] = 0.f;
                        }
                        const float2 s = *reinterpret_cast<const float2*>(sc + c);
                        const float2 b = *reinterpret_cast<const float2*>(sc + F + c);
                        float v0 = fmaf(d[4 * k + 0], s.x, b.x), v1 = fmaf(d[4 * k + 1], s.y, b.y);
                        float v2 = fmaf(d[4 * k + 2], s.x, b.x), v3 = fmaf(d[4 * k + 3], s.y, b.y);
                        if (kConv2) {
                            const float4 r = rb[k % kResAhead];
                            if (k + kResAhead < 32) rb[k % kResAhead] = res[(k + kResAhead) * 256];
                            v0 += r.x; v1 += r.y; v2 += r.z; v3 += r.w;
                        }
                        if (kKeep || kLast) {
                            v0 = fmaxf(v0, 0.f); v1 = fmaxf(v1, 0.f); v2 = fmaxf(v2, 0.f); v3 = fmaxf(v3, 0.f);
                        }
                        if (!kLast) {
                            if (kKeep) res[k * 256] = make_float4(v0, v1, v2, v3);
                            const uint32_t h0 = pack_h2<!kKeep>(v0, v1);
                            const uint32_t h1 = pack_h2<!kKeep>(v2, v3);
                            const uint32_t off = t * 8 * kActSlot + (c >> 3) * C::kActCg;
                            asm volatile("st.shared.b32 [%0], %1;" ::"r"(act_row0 + off), "r"(h0) : "memory");
                            asm volatile("st.shared.b32 [%0], %1;" ::"r"(act_row0 + kActSlot + off), "r"(h1) : "memory");
                        } else {
                            const float4 w = *reinterpret_cast<const float4*>(hw + 2 * c);
                            const float2 wv = *reinterpret_cast<const float2*>(hw + 2 * F + c);
                            hs[0] = fmaf(v1, w.z, fmaf(v0, w.x, hs[0]));
                            hs[1] = fmaf(v1, w.w, fmaf(v0, w.y, hs[1]));
                            hs[2] = fmaf(v1, wv.y, fmaf(v0, wv.x, hs[2]));
                            hs[3] = fmaf(v3, w.z, fmaf(v2, w.x, hs[3]));
                            hs[4] = fmaf(v3, w.w, fmaf(v2, w.y, hs[4]));
                            hs[5] = fmaf(v3, wv.y, fmaf(v2, wv.x, hs[5]));
                            const int g = g0 + 8 * t, b = g % B, pix = (g / B) * 8 + x;
                            if (p.dbg_tower) {
                                if (pos0 + b < p.n)
                                    *reinterpret_cast<float2*>(p.dbg_tower + ((size_t)(pos0 + b) * 64 + pix) * F + c) = make_float2(v0, v1);
                                if (pos0 + b + 1 < p.n)
                                    *reinterpret_cast<float2*>(p.dbg_tower + ((size_t)(pos0 + b + 1) * 64 + pix) * F + c) = make_float2(v2, v3);
                            }
                            if (c == F - 8 + cq) {   // sub-tile t done: the four lanes of a quad hold disjoint channel sets of its rows
#pragma unroll
                                for (int h = 0; h < 6; ++h) {
                                    hs[h] += __shfl_xor_sync(0xffffffffu, hs[h], 1);
                                    hs[h] += __shfl_xor_sync(0xffffffffu, hs[h], 2);
                                }
                                const int q = lane & 3;
                                if (q < 2)   // lane q of the quad: board b + q
                                    store_head_features(feat_s + (b + q) * kHeadFeatures, ssh, pix, q ? hs[3] : hs[0], q ? hs[4] : hs[1],
                                                        q ? hs[5] : hs[2]);
                            }
                        }
                    }
                };
                using Conv2 = std::true_type;
                using NoConv2 = std::false_type;
                if (last) {
                    if (is_conv2) epilogue(Conv2(), std::integral_constant<int, kEpiLast>());
                    else epilogue(NoConv2(), std::integral_constant<int, kEpiLast>());
                } else if (is_conv2) {
                    epilogue(Conv2(), std::integral_constant<int, kEpiKeep>());
                } else if (keep_res) {
                    epilogue(NoConv2(), std::integral_constant<int, kEpiKeep>());
                } else {
                    epilogue(NoConv2(), std::integral_constant<int, kEpiRelu>());
                }
                if (!last) fence_proxy_async();
            }
            // the tile's head features, staged in shared memory by the last epilogue (global stores there cost spills)
            epi_bar();
            if (pos0 < p.n) {
                const uint32_t nf = (p.n - pos0 < (uint32_t)B ? p.n - pos0 : (uint32_t)B) * kHeadFeatures;
                for (uint32_t i = et; i < nf; i += 256) p.feat[(size_t)pos0 * kHeadFeatures + i] = feat_s[i];
            }
        }
    }

    __syncthreads();
    if (CL > 1) cluster_sync_all();
}

}  // namespace narrow

int launch_tower_narrow(const Params& p, int filters, cudaStream_t stream) {
    using narrow::Cfg;
    using narrow::net_tower_narrow_kernel;
    if (filters == 128)
        return launch_tower_pairs<net_tower_narrow_kernel<128, 1>, net_tower_narrow_kernel<128, 2>, Cfg<128>::kSmemAlloc, Cfg<128>::B>(
            p, stream);
    return launch_tower_pairs<net_tower_narrow_kernel<64, 1>, net_tower_narrow_kernel<64, 2>, Cfg<64>::kSmemAlloc, Cfg<64>::B>(p, stream);
}

}  // namespace tc

}  // namespace rz
