// rz_tc_common.cuh -- PTX wrappers (mbarrier, bulk copy with cluster multicast, wgmma) and the pieces of the fused
// tower kernels that do not depend on their pipelines: parameter block, CTA-pair launch, layer-0 operand, head features.
#pragma once
#include <cuda_fp16.h>
#include "rz_bitboard.cuh"
#include "rz_net.cuh"

namespace rz {
namespace tc {

// ---- PTX wrappers ---------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
// arrive on the barrier at the same offset in CTA `rank` of the cluster
__device__ __forceinline__ void mbar_arrive_cta(uint32_t bar, uint32_t rank) {
    uint32_t remote;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(remote) : "r"(bar), "r"(rank));
    asm volatile("mbarrier.arrive.shared::cluster.b64 _, [%0];" ::"r"(remote) : "memory");
}
// Bounded wait (~4 s of SM clocks): a protocol bug traps and is reported to the host instead of hanging the GPU.
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
    uint32_t ok = 0;
    long long t0 = 0;
    for (uint32_t spin = 0; !ok; ++spin) {
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t}"
            : "=r"(ok)
            : "r"(bar), "r"(parity)
            : "memory");
        if (!ok && (spin & 1023) == 1023) {
            const long long now = clock64();
            if (t0 == 0) t0 = now;
            else if (now - t0 > 8000000000LL) __trap();
        }
    }
}
__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst), "l"(src),
                 "r"(bytes), "r"(bar)
                 : "memory");
}
// multicast variant (thread-block cluster): the copy lands at the same CTA-relative offset in every CTA of `mask` and
// signals the mbarrier at the same offset there
__device__ __forceinline__ void bulk_g2s_mc(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar, uint16_t mask) {
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster [%0], [%1], %2, [%3], %4;" ::"r"(dst),
        "l"(src), "r"(bytes), "r"(bar), "h"(mask)
        : "memory");
}
__device__ __forceinline__ void cluster_sync_all() {
    asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
__device__ __forceinline__ uint32_t cluster_ctarank() {
    uint32_t r;
    asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
    return r;
}
// 4-byte global -> shared copy that needs no register (LDGSTS); cp_async_wait_all() waits for this thread's copies
__device__ __forceinline__ void cp_async_4(uint32_t dst, const void* src) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(dst), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_all;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
// named barrier of the 256 math threads (warps 0..7)
__device__ __forceinline__ void epi_bar() { asm volatile("bar.sync 1, 256;" ::: "memory"); }

// wgmma shared-memory matrix descriptor: K-major, no swizzle; core matrix = 8 rows x 16 B (rows 16 B apart);
// LBO = byte distance between core matrices adjacent in K, SBO = byte distance between 8-row groups.
__device__ __forceinline__ uint64_t smem_desc(uint32_t addr, uint32_t lbo, uint32_t sbo) {
    return (uint64_t)((addr >> 4) & 0x3FFF) | ((uint64_t)((lbo >> 4) & 0x3FFF) << 16) | ((uint64_t)((sbo >> 4) & 0x3FFF) << 32);
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// pins the accumulator registers at this point of the instruction stream (no use or definition moves across)
__device__ __forceinline__ void acc_fence(float (&d)[128]) {
#pragma unroll
    for (int i = 0; i < 128; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

#define RZ_D4(i) "+f"(d[i]), "+f"(d[i + 1]), "+f"(d[i + 2]), "+f"(d[i + 3])
#define RZ_D16(i) RZ_D4(i), RZ_D4(i + 4), RZ_D4(i + 8), RZ_D4(i + 12)
// D[64 x 256] (+)= A[64 x 16] * B[16 x 256]: fp16 operands from shared memory (both K-major), fp32 accumulators in
// registers; accumulate = 0 overwrites D.
__device__ __forceinline__ void wgmma_m64n256k16(float (&d)[128], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %130, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n256k16.f32.f16.f16 {"
        "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
        "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
        "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, "
        "%64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, "
        "%80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, "
        "%96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, "
        "%112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127"
        "}, %128, %129, p, 1, 1, 0, 0;\n\t}"
        : RZ_D16(0), RZ_D16(16), RZ_D16(32), RZ_D16(48), RZ_D16(64), RZ_D16(80), RZ_D16(96), RZ_D16(112)
        : "l"(adesc), "l"(bdesc), "r"(accumulate)
        : "memory");
}
// narrower N for the 64- / 128-filter tower (rz_net_tc_narrow.cu): D = d[O .. O + N/2 - 1] of the thread's 128 accumulators,
// so that 256 / N such MMAs of one warpgroup (different A rows, the same B) fill the same register array
template <int O>
__device__ __forceinline__ void wgmma_m64n128k16(float (&d)[128], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 {"
        "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
        "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
        "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63"
        "}, %64, %65, p, 1, 1, 0, 0;\n\t}"
        : RZ_D16(O), RZ_D16(O + 16), RZ_D16(O + 32), RZ_D16(O + 48)
        : "l"(adesc), "l"(bdesc), "r"(accumulate)
        : "memory");
}
template <int O>
__device__ __forceinline__ void wgmma_m64n64k16(float (&d)[128], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %34, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {"
        "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31"
        "}, %32, %33, p, 1, 1, 0, 0;\n\t}"
        : RZ_D16(O), RZ_D16(O + 16)
        : "l"(adesc), "l"(bdesc), "r"(accumulate)
        : "memory");
}
#undef RZ_D16
#undef RZ_D4

// two fp32 -> packed fp16x2 (a in the low half), saturating at +-65504; RELU folds max(x, 0) into the convert
template <bool RELU>
__device__ __forceinline__ uint32_t pack_h2(float a, float b) {
    uint32_t d;
    if (RELU) asm("cvt.rn.relu.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(d) : "f"(b), "f"(a));
    else      asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(d) : "f"(b), "f"(a));
    return d;
}

struct Params {
    const __half* w0;   // layer-0 weight image (16 KB)
    const __half* w;    // tower weight stages
    const float* ss;    // folded BN [L][2][256], then heads
    const float* blob;  // fp32 blob for the head weights
    size_t off_policy_conv, off_policy_fc_k, off_policy_fc_b, off_value_conv, off_value_fc1_k, off_value_fc1_b, off_value_fc2_k,
        off_value_fc2_b;
    const u64* own;
    const u64* enemy;
    float* policy;
    float* value;
    float* res;        // fp32 residual stream, [CTA][32][256 threads][4]
    float* feat;       // head features, [n][kHeadFeatures]: written by the tower, read by the head pass
    float* dbg_tower;  // nullable
    float* dbg_logits; // nullable: [n][64] policy logits (before the softmax)
    float* dbg_vlogit; // nullable: [n] value before the tanh
    uint32_t n;
    const uint32_t* n_dev;  // nullable: batch size produced on the device (engine waves)
    int n_layers;  // 1 + 2R
    int V;
};

constexpr uint32_t kTcMaxV = 512;

// threads of the throughput towers: warps 0..7 = two math warpgroups, warps 8..11 = producer warpgroup
constexpr int kThreads = 384;

// Launches a throughput tower over the tiles of p.n boards, kBoards per tile: K2 in CTA pairs that share every weight
// stage (tower_cluster() == 2, where the GPU can hold a pair), else K1 in single CTAs.  grid = min(tiles, SMs); for pairs
// it is rounded up to whole clusters (a surplus CTA runs dummy tiles) and capped at the pairs the GPU holds at once.
// Callers hold the tower lock (rz_net.cu), which also guards the one-time setup.
template <void (*K1)(Params), void (*K2)(Params), uint32_t kSmem, uint32_t kBoards>
int launch_tower_pairs(const Params& p, cudaStream_t stream) {
    static int max_pairs = -1;
    if (max_pairs < 0) {
        RZ_CUDA_TRY(cudaFuncSetAttribute(K1, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmem));
        RZ_CUDA_TRY(cudaFuncSetAttribute(K2, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmem));
        // how many CTA pairs can be resident at once: an SM without a free partner in its GPC cannot take a pair
        cudaLaunchConfig_t cfg = {};
        cfg.gridDim = dim3((unsigned)num_sms() & ~1u); cfg.blockDim = dim3(kThreads); cfg.dynamicSmemBytes = kSmem;
        cudaLaunchAttribute attr[1];
        attr[0].id = cudaLaunchAttributeClusterDimension;
        attr[0].val.clusterDim.x = 2; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
        cfg.attrs = attr; cfg.numAttrs = 1;
        RZ_CUDA_TRY(cudaOccupancyMaxActiveClusters(&max_pairs, K2, &cfg));
    }
    const int cluster = tower_cluster() == 2 && max_pairs >= 1 ? 2 : 1;
    const uint32_t ntiles = (p.n + kBoards - 1) / kBoards;
    uint32_t grid = ntiles < (uint32_t)num_sms() ? ntiles : (uint32_t)num_sms();
    if (cluster == 1) {
        K1<<<grid, kThreads, kSmem, stream>>>(p);
    } else {
        grid = (grid + 1) & ~1u;
        if (grid > 2u * (uint32_t)max_pairs) grid = 2u * (uint32_t)max_pairs;
        cudaLaunchConfig_t cfg = {};
        cfg.gridDim = dim3(grid); cfg.blockDim = dim3(kThreads); cfg.dynamicSmemBytes = kSmem; cfg.stream = stream;
        cudaLaunchAttribute attr[1];
        attr[0].id = cudaLaunchAttributeClusterDimension;
        attr[0].val.clusterDim.x = 2; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
        cfg.attrs = attr; cfg.numAttrs = 1;
        RZ_CUDA_TRY(cudaLaunchKernelEx(&cfg, K2, p));
    }
    RZ_LAUNCH_CHECK();
    return RZ_OK;
}

// the tower families' launches on p.n boards, under the tower lock: 256 filters in 2-board tiles (rz_net_tc.cu); 64 and
// 128 filters in 512 / F-board tiles (rz_net_tc_narrow.cu); 256 filters with every 2-board tile on an 8-CTA cluster
// (rz_net_split.cu)
int launch_tower(const Params& p, cudaStream_t stream);
int launch_tower_narrow(const Params& p, int filters, cudaStream_t stream);
int launch_tower_split(const Params& p, cudaStream_t stream);

// layer-0 operand (agent/model.py:30-33 first convolution as a GEMM): im2col of the two bit planes of one board row m =
// (g, x), K index = tap * 2 + plane padded to 32, two of the four 8-wide K chunks (kc0, kc0 + 1) per calling thread;
// a0 = the [4 kc][16 g][8 x][8] fp16 tile in shared memory
__device__ __forceinline__ void build_layer0_operand(uint8_t* a0, u64 o, u64 e, int kc0, int g, int x, int y) {
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
        *reinterpret_cast<uint4*>(a0 + kc * 2048 + g * 128 + x * 16) = make_uint4(w[0], w[1], w[2], w[3]);
    }
}

// head features of one pixel of one board: BN + ReLU of its 1x1 head-conv sums (policy filters 0, 1 and value), stored
// to the board's row f of the head-feature buffer in the Flatten (C,H,W) order of agent/model.py: policy c*64 + pix,
// value 128 + pix.  The dense heads run on them afterwards, batched over all boards (rz_net_heads.cu).
__device__ __forceinline__ void store_head_features(float* f, const float* ssh, int pix, float a0, float a1, float av) {
    f[pix] = fmaxf(fmaf(a0, ssh[0], ssh[2]), 0.f);
    f[64 + pix] = fmaxf(fmaf(a1, ssh[1], ssh[3]), 0.f);
    f[128 + pix] = fmaxf(fmaf(av, ssh[4], ssh[5]), 0.f);
}

}  // namespace tc

// the dense heads after a tower (rz_net_heads.cu): Dense(128 -> 64) + softmax and Dense(64 -> V) + ReLU -> Dense(V -> 1) +
// tanh over p.feat for p.n boards (p.n_dev when set), many boards per CTA, on the tower's stream
int net_heads(const tc::Params& p, cudaStream_t stream);

}  // namespace rz
