// rz_net_tc.cu -- K4/K5: fused persistent wgmma residual tower + head features for the 256-filter network (sm_90a).
//
// One CTA per SM, each CTA owns a tile of TWO boards (M = 128 pixel rows) and carries it through the
// WHOLE network without writing activations to HBM in between:
//   * activations live in shared memory as fp16 in the wgmma "K-major, no-swizzle" canonical layout,
//     with a one-pixel zero border, so that each of the nine 3x3 taps is just a different start
//     address of the same buffer (implicit GEMM, no im2col copy):
//         chunk(cg, slot, xp) at cg*2896 + slot*144 + xp*16 bytes   (8 channels = 16 B per chunk)
//         slot = 2*(y+1) + board (the two boards' rows are interleaved so that a dy shift is a
//         uniform 2-slot offset), xp = x+1; xp = 9 of one slot aliases xp = 0 of the next (shared
//         zero chunk).  MMA row m = (2y+board)*8 + x  ->  8-row core matrices are board rows.
//   * weights (fp16, 1.18 MB per conv, L2-resident) are streamed by a producer warp with
//     cp.async.bulk in pre-packed 32 KB stages (one tap x 64 input channels x 256 output channels)
//     through a 3-deep mbarrier ring; with clusters of two CTAs each CTA fetches half of every stage
//     and multicasts it into both CTAs' shared memory, which halves the L2 -> SM weight traffic;
//   * two math warpgroups, one per 64 rows (the rows y = 0-3 / 4-7 of both boards), issue
//     wgmma.m64n256k16 (fp16 in / fp32 accumulate in registers): 144 per conv layer and warpgroup;
//   * the same warpgroups then apply the folded BatchNorm (scale, shift), the skip connection and
//     ReLU to their accumulators and write the next layer's fp16 activations straight back into the
//     shared-memory operand buffer.  The fp32 residual stream (the block inputs) does not fit beside
//     the accumulators in the register file, nor beside the operands in shared memory; it goes to a
//     per-CTA global scratch of the network (128 KB, written once and read once per block, L2-resident);
//   * the epilogue does not wait on L2 one load at a time: a conv2 layer's first residual loads are issued before its
//     last wgmma_wait and every later one kResAhead steps before its use; each layer's BN scale / shift is copied
//     (cp.async) into the idle half of a double buffer while the previous layer's MMAs run; the 1x1 head-conv weights
//     are staged in shared memory once per CTA;
//   * the first conv (2 -> 256 channels, K = 18 padded to 32) is a 2-MMA GEMM on an im2col tile built
//     from the two bitboards; the last epilogue reduces the fp32 tower output to the 1x1 head convolutions and stores
//     their BN + ReLU outputs (192 fp32 per board) for the dense heads, which run afterwards as one batched pass over
//     all boards (rz_net_heads.cu) instead of once per tile on the math warps.
// Global traffic per position: 16 B in and 768 B of head features out (the head pass reads them back and writes the
// 260 B of policy and value).  Algorithmic work: 2 * 755,343,616 flop (SURVEY 3.2).
// Host side: launch_tower, a CTA-pair launch (launch_tower_pairs, rz_tc_common.cuh) called by the one tower sequence of
// all three tower families (tower_forward, rz_net.cu).  rz_net.cu also packs the weight image at load (tc_w, rz_net.cuh).
#include <stdlib.h>
#include <type_traits>
#include "rz_bitboard.cuh"
#include "rz_net.cuh"
#include "rz_tc_common.cuh"

namespace rz {
namespace tc {

// kThreads = 384: warps 0..7 = two math warpgroups, warps 8..11 = producer warpgroup (one thread streams the weights).
// Registers are handed from the producer warpgroup to the math warpgroups (setmaxnreg): the math threads hold a 64 x 256
// fp32 accumulator (128 registers) each.
constexpr uint32_t kProducerRegs = 40, kMathRegs = 232;
constexpr int kMathThreads = 256;
constexpr uint32_t kActCg = 2896, kActSlot = 144;
constexpr uint32_t kActBytes = 32 * kActCg;  // 92,672
constexpr uint32_t kStageBytes = 32768, kStages = 3;
constexpr int kResAhead = 4;   // residual float4 loads a conv2 epilogue keeps in flight (16 registers; 8 would spill)
constexpr uint32_t kA0Bytes = 8192, kW0Bytes = 16384;
constexpr uint32_t kOffAct = 0;
constexpr uint32_t kOffW = kOffAct + kActBytes;
constexpr uint32_t kOffA0 = kOffW + kStages * kStageBytes;
constexpr uint32_t kOffW0 = kOffA0 + kA0Bytes;
constexpr uint32_t kOffSS = kOffW0 + kW0Bytes;           // 2 x [scale 256][shift 256] fp32
constexpr uint32_t kOffHw = kOffSS + 2 * 2048;           // 1x1 head-conv weights: policy [256][2], value [256] fp32
constexpr uint32_t kOffBar = kOffHw + 768 * 4;           // mbarriers
constexpr uint32_t kNumBars = 2 * kStages + 1;           // full[], empty[], w0
constexpr uint32_t kSmemBytes = kOffBar + kNumBars * 8;
constexpr uint32_t kSmemAlloc = kSmemBytes + 128;  // slack for manual 128 B alignment
static_assert(kSmemAlloc <= 232448, "shared memory budget exceeded");
static_assert(kTowerResFloatsPerCta == (size_t)kMathThreads * 128, "residual scratch per CTA");

// Phase stamps (build with -DRZ_TOWER_STAMPS; tools/tower_phases.py): SM-clock deltas summed per CTA into
// g_tower_stamps[blockIdx.x][phase], as seen by math thread 0 (warpgroup 0) and, for kStEmpty, by the producer thread.
// Off by default: RZ_STAMP(...) expands to nothing and the production kernel is compiled as if the stamps did not exist.
#ifdef RZ_TOWER_STAMPS
enum : int {
    kStTiles,    // tiles processed (a count, not cycles)
    kStTile,     // whole tile, layer-0 operand to the last head-feature store
    kStKLoop,    // MMA sections of all layers: from the first weight wait to the last wgmma_wait
    kStFull,     // waiting on bar_full (weights late; the wgmmas already queued keep running meanwhile)
    kStMma,      // waiting in wgmma_wait (MMA-bound)
    kStEpiBar,   // waiting at epi_bar around the layer boundaries
    kStEpi0,     // layer-0 epilogue
    kStEpi1,     // conv1 epilogues (first conv of a block)
    kStEpi2,     // conv2 epilogues (second conv of a block), except the last layer's
    kStEpiLast,  // last layer's epilogue (head 1x1 sums)
    kStFeat,     // head features: the 1x1 sums reduced over the lane quad, BN + ReLU, stored to global memory
    kStEmpty,    // producer: waiting on bar_empty (slot not yet released by both CTAs' math warps)
    kStCount
};
constexpr int kStMaxCtas = 1024;
__device__ unsigned long long g_tower_stamps[kStMaxCtas][kStCount];
__device__ __forceinline__ void stamp_add(int phase, uint32_t cycles) { atomicAdd(&g_tower_stamps[blockIdx.x][phase], (unsigned long long)cycles); }
#define RZ_STAMP(...) __VA_ARGS__
#else
#define RZ_STAMP(...)
#endif

// CL = thread-block-cluster size (1 or 2).  With CL = 2 the two CTAs of a cluster each fetch half of every weight
// stage from L2 and multicast it into both CTAs' shared memory; MMAs and the epilogue stay per-CTA.  A stage may be
// refilled only after BOTH CTAs' math warps have read it, so the `empty` barriers count the arrivals of 8 warps per CTA.
template <int CL>
__global__ void __launch_bounds__(kThreads, 1) net_tower_kernel(const Params pp) {
    Params p = pp;
    if (p.n_dev) p.n = *p.n_dev;
    extern __shared__ uint8_t smem_raw[];
    const uint32_t base = (smem_u32(smem_raw) + 127u) & ~127u;
    uint8_t* sm = smem_raw + (base - smem_u32(smem_raw));
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t bar0 = base + kOffBar;
    auto bar_full = [&](uint32_t s) { return bar0 + s * 8; };
    auto bar_empty = [&](uint32_t s) { return bar0 + (kStages + s) * 8; };
    const uint32_t bar_w0 = bar0 + 2 * kStages * 8;
    const uint32_t ntiles = (p.n + 1) >> 1;
    const int L = p.n_layers;
    // every CTA of a cluster runs the same number of tile iterations (the producers are coupled through the shared
    // weight ring); a CTA whose last tile index is past the batch processes an all-empty dummy tile
    const uint32_t crank = CL > 1 ? cluster_ctarank() : 0u;
    const uint32_t cbase = blockIdx.x - crank;
    const uint32_t iters = cbase < ntiles ? (ntiles - cbase + gridDim.x - 1) / gridDim.x : 0u;

    // ---- one-time setup -----------------------------------------------------------------------------
    for (uint32_t i = threadIdx.x * 16; i < kActBytes; i += kThreads * 16) *reinterpret_cast<uint4*>(sm + kOffAct + i) = make_uint4(0, 0, 0, 0);
    fence_proxy_async();
    // the 1x1 head-conv weights are the same for every tile: staged once, read from shared memory by the last epilogue
    for (uint32_t i = threadIdx.x; i < 768; i += kThreads)
        reinterpret_cast<float*>(sm + kOffHw)[i] = __ldg(i < 512 ? p.blob + p.off_policy_conv + i : p.blob + p.off_value_conv + (i - 512));
    if (threadIdx.x == 0) {
        for (uint32_t s = 0; s < kStages; ++s) { mbar_init(bar_full(s), 1); mbar_init(bar_empty(s), 8 * CL); }
        mbar_init(bar_w0, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    if (CL > 1) cluster_sync_all();  // peers' barriers are initialised before anyone multicasts into them

    if (warp >= 8) {
        // ===== weight producer =====================================================================
        asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(kProducerRegs));
        if (warp == 8 && lane == 0) {
            if (iters > 0) {   // a CTA without tiles must not leave with a copy into its shared memory in flight
                mbar_expect_tx(bar_w0, kW0Bytes);
                bulk_g2s(base + kOffW0, p.w0, kW0Bytes, bar_w0);
            }
            uint32_t stage = 0, phase = 0;
            for (uint32_t it = 0; it < iters; ++it) {
                for (int l = 1; l < L; ++l) {
                    const uint8_t* src = reinterpret_cast<const uint8_t*>(p.w) + (size_t)(l - 1) * 36 * kStageBytes;
                    RZ_STAMP(uint32_t st_empty = 0;)
                    for (int s = 0; s < 36; ++s) {
                        RZ_STAMP(const uint32_t c0 = (uint32_t)clock();)
                        mbar_wait(bar_empty(stage), phase ^ 1);
                        RZ_STAMP(st_empty += (uint32_t)clock() - c0;)
                        mbar_expect_tx(bar_full(stage), kStageBytes);
                        if (CL == 1) {
                            bulk_g2s(base + kOffW + stage * kStageBytes, src + (size_t)s * kStageBytes, kStageBytes, bar_full(stage));
                        } else {  // this CTA's slice of the stage, delivered to every CTA of the cluster
                            constexpr uint32_t kSlice = kStageBytes / CL;
                            bulk_g2s_mc(base + kOffW + stage * kStageBytes + crank * kSlice, src + (size_t)s * kStageBytes + crank * kSlice,
                                        kSlice, bar_full(stage), (uint16_t)((1u << CL) - 1u));
                        }
                        if (++stage == kStages) { stage = 0; phase ^= 1; }
                    }
                    RZ_STAMP(stamp_add(kStEmpty, st_empty);)
                }
            }
        }
    } else {
        // ===== math warpgroups (2) =================================================================
        asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(kMathRegs));
        const int et = threadIdx.x;           // 0..255
        const int wg = warp >> 2;             // rows wg*64 .. wg*64 + 63
        // accumulator fragment of wgmma m64n256: d[4i + 0/1] = row r0, columns c, c + 1; d[4i + 2/3] = row r0 + 8;
        // c = 8i + 2 (lane & 3).  Rows r0 and r0 + 8 are the same pixel (y, x) of board 0 and board 1.
        const int r0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);
        const int g0 = r0 >> 3, x = r0 & 7, y = g0 >> 1;
        const int cq = 2 * (lane & 3);
        const uint32_t act_row0 = base + kOffAct + (g0 + 2) * kActSlot + (x + 1) * 16 + cq * 2;  // + cg * kActCg
        const uint32_t act_row1 = act_row0 + kActSlot;
        const uint32_t a_wg = base + kOffAct + wg * 8 * kActSlot;   // operand rows of this warpgroup, tap (0, 0)
        float* ss_s = reinterpret_cast<float*>(sm + kOffSS);
        float4* res = reinterpret_cast<float4*>(p.res + (size_t)blockIdx.x * kTowerResFloatsPerCta) + et;   // + i * 256
        const float* hw = reinterpret_cast<const float*>(sm + kOffHw);
        uint32_t stage = 0, phase = 0, ss_buf = 0;
        float d[128];
        // BN parameters of the first layer; every later layer's are fetched one layer ahead (below)
        ss_s[et] = __ldg(p.ss + et);
        ss_s[256 + et] = __ldg(p.ss + 256 + et);

        for (uint32_t it = 0; it < iters; ++it) {
            const uint32_t tile = blockIdx.x + it * gridDim.x;  // may be >= ntiles: dummy tile (no valid board)
            const uint32_t pos0 = tile * 2;
            RZ_STAMP(const uint32_t st_tile0 = (uint32_t)clock();)
            {   // ---- layer-0 operand: im2col of the two bit planes, K index = tap*2 + plane, padded to 32 ----
                const int m = et & 127, g = m >> 3, brd = g & 1;
                const bool valid = pos0 + brd < p.n;
                build_layer0_operand(sm + kOffA0, valid ? p.own[pos0 + brd] : 0, valid ? p.enemy[pos0 + brd] : 0, 2 * (et >> 7), g, m & 7,
                                     g >> 1);
                fence_proxy_async();
            }
            float hs[6];   // head partial sums (policy 0, policy 1, value) x (board 0, 1): set by the last epilogue only, so that
                           // they do not hold registers through the K loops
            for (int l = 0; l < L; ++l) {
                // folded BN parameters, double-buffered across layers: this layer's were copied in during the previous
                // layer; the next layer's (after the last layer: the first layer's, for the next tile) are copied into
                // the other buffer while this layer's MMAs run, so no layer starts on an L2 read
                const float* sc = ss_s + ss_buf * 512;
                const bool is_conv2 = l > 0 && (l & 1) == 0;   // second conv of a block: add the skip connection
                float4 rb[kResAhead];   // residual loads in flight (conv2 layers)
                RZ_STAMP(uint32_t st_c = (uint32_t)clock(), st_bar = 0, st_full = 0, st_mma = 0;)
                epi_bar();   // operand (written by both warpgroups, made visible to the async proxy) and BN params ready;
                             // every thread is done with layer l - 1's epilogue, so the other BN buffer is free
                RZ_STAMP(st_bar += (uint32_t)clock() - st_c;)
                {
                    const size_t nl = l + 1 < L ? (size_t)l + 1 : 0;
                    const uint32_t dst = smem_u32(ss_s + (ss_buf ^ 1) * 512 + et);
                    cp_async_4(dst, p.ss + nl * 512 + et);
                    cp_async_4(dst + 1024, p.ss + nl * 512 + 256 + et);
                }
                RZ_STAMP(const uint32_t st_k0 = (uint32_t)clock();)
                acc_fence(d);
                if (l == 0) {
                    RZ_STAMP(st_c = (uint32_t)clock();)
                    mbar_wait(bar_w0, 0);
                    RZ_STAMP(st_full += (uint32_t)clock() - st_c;)
                    wgmma_fence();
#pragma unroll
                    for (uint32_t j = 0; j < 2; ++j)
                        wgmma_m64n256k16(d, smem_desc(base + kOffA0 + j * 2 * 2048 + wg * 1024, 2048, 128),
                                         smem_desc(base + kOffW0 + j * 2 * 4096, 4096, 128), j);
                    wgmma_commit();
                    RZ_STAMP(st_c = (uint32_t)clock();)
                    wgmma_wait<0>();
                    RZ_STAMP(st_mma += (uint32_t)clock() - st_c;)
                } else {
                    int prev = -1;
                    for (uint32_t tap = 0; tap < 9; ++tap) {
                        // tap (kh, kw) reads input pixel (y + kh - 1, x + kw - 1): slot offset 2*kh, chunk offset kw
                        const uint32_t a_tap = a_wg + (2 * (tap / 3)) * kActSlot + (tap % 3) * 16;
                        for (uint32_t kb = 0; kb < 4; ++kb) {
                            RZ_STAMP(st_c = (uint32_t)clock();)
                            mbar_wait(bar_full(stage), phase);
                            RZ_STAMP(st_full += (uint32_t)clock() - st_c;)
                            const uint32_t b_st = base + kOffW + stage * kStageBytes;
                            wgmma_fence();
#pragma unroll
                            for (uint32_t j = 0; j < 4; ++j)
                                wgmma_m64n256k16(d, smem_desc(a_tap + (kb * 8 + 2 * j) * kActCg, kActCg, kActSlot),
                                                 smem_desc(b_st + 2 * j * 4096, 4096, 128), (tap | kb | j) != 0);
                            wgmma_commit();
                            RZ_STAMP(st_c = (uint32_t)clock();)
                            wgmma_wait<1>();   // the previous stage's MMAs have completed: its slot may be refilled
                            RZ_STAMP(st_mma += (uint32_t)clock() - st_c;)
                            if (prev >= 0 && lane == 0) {
                                mbar_arrive(bar_empty(prev));
                                if (CL > 1) mbar_arrive_cta(bar_empty(prev), crank ^ 1u);
                            }
                            prev = (int)stage;
                            if (++stage == kStages) { stage = 0; phase ^= 1; }
                        }
                    }
                    // the first residual loads of the epilogue overlap the last stage's MMAs
                    if (is_conv2) {
#pragma unroll
                        for (int i = 0; i < kResAhead; ++i) rb[i] = res[i * 256];
                    }
                    RZ_STAMP(st_c = (uint32_t)clock();)
                    wgmma_wait<0>();
                    RZ_STAMP(st_mma += (uint32_t)clock() - st_c;)
                    if (lane == 0) {
                        mbar_arrive(bar_empty(prev));
                        if (CL > 1) mbar_arrive_cta(bar_empty(prev), crank ^ 1u);
                    }
                }
                RZ_STAMP(const uint32_t st_k1 = (uint32_t)clock();)
                acc_fence(d);
                cp_async_wait_all();   // the next layer's BN parameters have landed (published by the next barrier)
                ss_buf ^= 1;
                const bool keep_res = l == 0 || is_conv2;      // block output: keep an fp32 copy for the skip connection
                const bool last = l == L - 1;
                RZ_STAMP(st_c = (uint32_t)clock();)
                if (!last) epi_bar();   // both warpgroups' MMAs have finished reading the operand it is about to overwrite
                RZ_STAMP(const uint32_t st_e0 = (uint32_t)clock(); st_bar += st_e0 - st_c;)
                float* dbg0 = nullptr;
                float* dbg1 = nullptr;
                if (last && p.dbg_tower) {
                    if (pos0 < p.n) dbg0 = p.dbg_tower + ((size_t)pos0 * 64 + y * 8 + x) * 256;
                    if (pos0 + 1 < p.n) dbg1 = p.dbg_tower + ((size_t)(pos0 + 1) * 64 + y * 8 + x) * 256;
                }
                // the epilogue is compiled once per layer kind, so that its unrolled loop holds no branch: the compiler
                // can then hoist the BN loads and interleave the steps, and a conv2 layer's residual loads land straight
                // in the registers that consume them kResAhead steps later.  kConv2: add the skip connection; kKind:
                // kEpiRelu (first conv of a block: ReLU folded into the fp16 convert), kEpiKeep (block output: ReLU, fp32
                // copy kept for the skip connection), kEpiLast (tower output: ReLU, head 1x1 sums)
                constexpr int kEpiRelu = 0, kEpiKeep = 1, kEpiLast = 2;
                auto epilogue = [&](auto conv2, auto kind) {
                    constexpr bool kConv2 = decltype(conv2)::value;
                    constexpr bool kKeep = decltype(kind)::value == kEpiKeep, kLast = decltype(kind)::value == kEpiLast;
                    if (kLast) {
#pragma unroll
                        for (int k = 0; k < 6; ++k) hs[k] = 0.f;
                    }
#pragma unroll
                for (int i = 0; i < 32; ++i) {
                    const int c = 8 * i + cq;
                    const float2 s = *reinterpret_cast<const float2*>(sc + c);
                    const float2 b = *reinterpret_cast<const float2*>(sc + 256 + c);
                    float v0 = fmaf(d[4 * i + 0], s.x, b.x), v1 = fmaf(d[4 * i + 1], s.y, b.y);
                    float v2 = fmaf(d[4 * i + 2], s.x, b.x), v3 = fmaf(d[4 * i + 3], s.y, b.y);
                    if (kConv2) {   // step i's residual was loaded kResAhead steps earlier; its slot takes step i + kResAhead's
                        const float4 r = rb[i % kResAhead];
                        if (i + kResAhead < 32) rb[i % kResAhead] = res[(i + kResAhead) * 256];
                        v0 += r.x; v1 += r.y; v2 += r.z; v3 += r.w;
                    }
                    if (kKeep || kLast) {
                        v0 = fmaxf(v0, 0.f); v1 = fmaxf(v1, 0.f); v2 = fmaxf(v2, 0.f); v3 = fmaxf(v3, 0.f);
                    }
                    if (!kLast) {
                        if (kKeep) res[i * 256] = make_float4(v0, v1, v2, v3);
                        const uint32_t h0 = pack_h2<!kKeep>(v0, v1);
                        const uint32_t h1 = pack_h2<!kKeep>(v2, v3);
                        const uint32_t off = (c >> 3) * kActCg;
                        asm volatile("st.shared.b32 [%0], %1;" ::"r"(act_row0 + off), "r"(h0) : "memory");
                        asm volatile("st.shared.b32 [%0], %1;" ::"r"(act_row1 + off), "r"(h1) : "memory");
                    } else {  // tower output feeds the 1x1 head convolutions (policy: 2 filters, value: 1)
                        const float4 w = *reinterpret_cast<const float4*>(hw + 2 * c);   // policy filters 0, 1 of c, c + 1
                        const float2 wv = *reinterpret_cast<const float2*>(hw + 512 + c);
                        hs[0] = fmaf(v1, w.z, fmaf(v0, w.x, hs[0]));
                        hs[1] = fmaf(v1, w.w, fmaf(v0, w.y, hs[1]));
                        hs[2] = fmaf(v1, wv.y, fmaf(v0, wv.x, hs[2]));
                        hs[3] = fmaf(v3, w.z, fmaf(v2, w.x, hs[3]));
                        hs[4] = fmaf(v3, w.w, fmaf(v2, w.y, hs[4]));
                        hs[5] = fmaf(v3, wv.y, fmaf(v2, wv.x, hs[5]));
                        if (dbg0) *reinterpret_cast<float2*>(dbg0 + c) = make_float2(v0, v1);
                        if (dbg1) *reinterpret_cast<float2*>(dbg1 + c) = make_float2(v2, v3);
                    }
                }
                };
                using Conv2 = std::true_type;
                using NoConv2 = std::false_type;
                if (last) {
                    if (is_conv2) epilogue(Conv2(), std::integral_constant<int, kEpiLast>());
                    else epilogue(NoConv2(), std::integral_constant<int, kEpiLast>());   // no residual block: layer 0 is last
                } else if (is_conv2) {
                    epilogue(Conv2(), std::integral_constant<int, kEpiKeep>());
                } else if (keep_res) {
                    epilogue(NoConv2(), std::integral_constant<int, kEpiKeep>());     // layer 0
                } else {
                    epilogue(NoConv2(), std::integral_constant<int, kEpiRelu>());
                }
                if (!last) fence_proxy_async();
                RZ_STAMP(if (et == 0) {
                    stamp_add(kStKLoop, st_k1 - st_k0); stamp_add(kStFull, st_full); stamp_add(kStMma, st_mma); stamp_add(kStEpiBar, st_bar);
                    stamp_add(l == 0 ? kStEpi0 : last ? kStEpiLast : is_conv2 ? kStEpi2 : kStEpi1, (uint32_t)clock() - st_e0);
                })
            }
            RZ_STAMP(const uint32_t st_h0 = (uint32_t)clock();)
            // ---- head features (agent/model.py:43-47) of the tile's two boards -----------------------------------
            // the four lanes of a row quad hold disjoint column sets of the same two rows; lane q < 2 stores board q's features
#pragma unroll
            for (int k = 0; k < 6; ++k) {
                hs[k] += __shfl_xor_sync(0xffffffffu, hs[k], 1);
                hs[k] += __shfl_xor_sync(0xffffffffu, hs[k], 2);
            }
            {
                const int q = lane & 3;
                if (q < 2 && pos0 + q < p.n) {
                    // constant indices keep hs in registers (a lane-dependent index would put it in local memory).  The
                    // + 0.f is the second column half's (zero) partial sum of the reduction these features were first
                    // computed with; it turns a -0 sum into +0, and the outputs are held to those bits
                    const float h0 = q ? hs[3] : hs[0], h1 = q ? hs[4] : hs[1], h2 = q ? hs[5] : hs[2];
                    store_head_features(p.feat + (size_t)(pos0 + q) * kHeadFeatures, p.ss + (size_t)L * 512, y * 8 + x, h0 + 0.f,
                                        h1 + 0.f, h2 + 0.f);
                }
            }
            RZ_STAMP(if (et == 0) {
                const uint32_t st_h1 = (uint32_t)clock();
                stamp_add(kStFeat, st_h1 - st_h0); stamp_add(kStTile, st_h1 - st_tile0); stamp_add(kStTiles, 1);
            })
        }
    }

    __syncthreads();
    if (CL > 1) cluster_sync_all();  // no CTA leaves while a peer may still multicast into it / arrive on its barriers
}

int launch_tower(const Params& p, cudaStream_t stream) {
    return launch_tower_pairs<net_tower_kernel<1>, net_tower_kernel<2>, kSmemAlloc, 2>(p, stream);
}

}  // namespace tc

static int g_cluster = 0;        // 0: not yet decided (RZ_TOWER_CLUSTER, default 2)

int set_tower_cluster(int cluster) {
    RZ_REQUIRE(cluster == 1 || cluster == 2, "rz_net_set_tower_cluster: cluster must be 1 or 2");
    g_cluster = cluster;
    return RZ_OK;
}

int tower_cluster() {
    if (g_cluster == 0) {
        const char* cs = getenv("RZ_TOWER_CLUSTER");
        g_cluster = (cs && atoi(cs) == 1) ? 1 : 2;
    }
    return g_cluster;
}

}  // namespace rz

#ifdef RZ_TOWER_STAMPS
// Stamped builds only (tools/tower_phases.py): copies the per-CTA phase sums, [n_ctas][kStCount] uint64, to `out`
// (when not null), then zeroes them if `reset`.  Returns a cudaError_t.
extern "C" int rz_tower_stamps(unsigned long long* out, int n_ctas, int reset) {
    using namespace rz::tc;
    if (n_ctas < 0 || n_ctas > kStMaxCtas) return (int)cudaErrorInvalidValue;
    const size_t bytes = (size_t)n_ctas * kStCount * sizeof(unsigned long long);
    cudaError_t e = cudaDeviceSynchronize();
    if (e == cudaSuccess && out) e = cudaMemcpyFromSymbol(out, g_tower_stamps, bytes);
    if (e == cudaSuccess && reset) {
        void* dev = nullptr;
        e = cudaGetSymbolAddress(&dev, g_tower_stamps);
        if (e == cudaSuccess) e = cudaMemset(dev, 0, sizeof(g_tower_stamps));
        if (e == cudaSuccess) e = cudaDeviceSynchronize();
    }
    return (int)e;
}
extern "C" int rz_tower_stamp_count() { return rz::tc::kStCount; }
#endif
