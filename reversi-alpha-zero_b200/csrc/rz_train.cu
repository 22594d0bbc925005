// rz_train.cu -- one SGD step of the policy/value network on the device (the reference's OptimizeWorker.train_epoch ->
// Keras fit on ReversiModel, agent/model.py:28-72,104-110, worker/optimize.py:73-86).
//
// Activations are fp32 NHWC [B*64 pixels][C] in device memory, layer by layer, because training-mode BatchNormalization
// needs the whole batch's conv output before it can normalise anything.  The 3x3 convolutions (forward, input gradient,
// weight gradient) run on tensor cores as TF32 mma.sync with fp32 accumulation; everything else is small CUDA-core
// kernels.  Every reduction has a fixed order (no floating-point atomics), so a step is bit-reproducible.
#include <math.h>
#include <stdlib.h>
#include <string.h>
#include <algorithm>
#include <new>
#include <type_traits>
#include <vector>
#include "rz_common.cuh"

namespace rz {
namespace {

constexpr float kTrainBnEps = 1e-3f;   // Keras BatchNormalization default epsilon
constexpr float kLogEps = 1e-7f;       // K.epsilon() inside the policy loss's log (agent/model.py:104-106)
constexpr int kCin0 = 16;              // conv0's 2 input planes, zero-padded to one GEMM k-chunk
constexpr int kRowsPerChunk = 64;      // column reductions: one partial per 64 pixels (= per record)
constexpr int kWgradTargetBlocks = 264;  // split-K of the weight gradient aims at 2 CTAs per SM on a 132-SM H100
constexpr int kUpdateBlocks = 512;     // fixed grid of the update kernel: its L2 partial sums have a fixed order

enum Kind : uint8_t { kKernel = 0, kTrainable = 1, kMovingMean = 2, kMovingVar = 3 };

// ---- TF32 implicit-GEMM convolution on mma.sync.m16n8k8 --------------------------------------------------------------
// CTA tile 128 x 128 x 16, 8 warps as 2 (M) x 4 (N), warp tile 64 x 32; operands staged through registers into a
// double-buffered shared-memory tile, rounded to TF32 (round to nearest, ties away) on the way.
//   kConv:  out[m][n] = sum_{tap, k} in[shift(m, tap)][k] * W[tap][k][n]  (+ bias[n]) (+ add[m][n])
//           M = B*64 pixels, N = Cout, K = 9*Cin; zero padding by mask.  Forward and input gradient (with the
//           mirrored, transposed weight image).
//   kWgrad: part[z][r][n] = sum_{m in split z} in[shift(m, tap(r))][ci(r)] * dy[m][n],  r = tap*Cin + ci
//           M = 9*Cin, N = Cout, K = pixels, split-K over blockIdx.z into scratch (reduced in a fixed order).
// mma.sync rather than wgmma: wgmma's TF32 form reads both operands K-major from shared memory, which neither
// backward GEMM has without a transpose; mma.sync takes fragments from any layout the loader chooses.
constexpr int kBM = 128, kBN = 128, kBK = 16;
constexpr int kAStr = kBK + 4;   // As[m][k] row stride (conflict-free fragment reads)
constexpr int kBStr = kBN + 8;   // Bs[k][n] and AsT[k][m] row stride

__device__ __forceinline__ uint32_t to_tf32(float x) {
    uint32_t r;
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
    return r;
}

__device__ __forceinline__ float4 tf32x4(float4 v) {
    return make_float4(__uint_as_float(to_tf32(v.x)), __uint_as_float(to_tf32(v.y)), __uint_as_float(to_tf32(v.z)),
                       __uint_as_float(to_tf32(v.w)));
}

__device__ __forceinline__ void mma_tf32(float* d, const uint32_t* a, const uint32_t* b) {
    asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}

// pixel m shifted by tap (dy, dx in -1..1); -1 when it falls off the board
__device__ __forceinline__ int shift_pixel(int m, int tap) {
    const int p = m & 63, y = (p >> 3) + tap / 3 - 1, x = (p & 7) + tap % 3 - 1;
    return (y < 0 || y > 7 || x < 0 || x > 7) ? -1 : (m & ~63) + y * 8 + x;
}

template <bool kWgrad>
__global__ void __launch_bounds__(256, 2)
conv_gemm_tf32_kernel(const float* __restrict__ in, int Cin, const float* __restrict__ B, int N, const float* __restrict__ bias,
                      const float* __restrict__ add, float* __restrict__ out, int M, int k_per_split) {
    // kConv: A = in (shifted gather), B = W[9*Cin][N], out [M][N].  kWgrad: A = in^T (rows r = tap*Cin+ci), B = dy [pixels][N].
    __shared__ __align__(16) float As[2][kWgrad ? kBK * kBStr : kBM * kAStr];
    __shared__ __align__(16) float Bs[2][kBK * kBStr];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int wm = warp & 1, wn = warp >> 1, g = lane >> 2, t4 = lane & 3;
    const int m0 = blockIdx.x * kBM, n0 = blockIdx.y * kBN;
    const int Mrows = kWgrad ? 9 * Cin : M;
    const int k_begin = kWgrad ? blockIdx.z * k_per_split : 0;
    const int k_total = kWgrad ? min(k_per_split, M - k_begin) : 9 * Cin;
    const int KT = k_total / kBK;

    float acc[4][4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j)
#pragma unroll
            for (int e = 0; e < 4; ++e) acc[i][j][e] = 0.f;

    float4 ra[2], rb[2];
    auto load = [&](int kt) {
        const int k0 = k_begin + kt * kBK;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int idx = tid + h * 256;
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (!kWgrad) {  // A[m][k]: 128 rows x 4 float4 along the channels of one tap
                const int row = idx >> 2, c4 = idx & 3, m = m0 + row;
                const int tap = k0 / Cin, c = k0 - tap * Cin + c4 * 4;
                const int src = m < M ? shift_pixel(m, tap) : -1;
                if (src >= 0) v = __ldg(reinterpret_cast<const float4*>(in + (size_t)src * Cin + c));
            } else {  // A^T[k = pixel][r]: 16 pixels x 32 float4 along the channels of one tap
                const int kk = idx >> 5, r = m0 + (idx & 31) * 4;
                if (r < Mrows) {
                    const int tap = r / Cin, c = r - tap * Cin;
                    const int src = shift_pixel(k0 + kk, tap);
                    if (src >= 0) v = __ldg(reinterpret_cast<const float4*>(in + (size_t)src * Cin + c));
                }
            }
            ra[h] = v;
            // B[k][n]: 16 rows x 32 float4
            const int kk = idx >> 5, n = n0 + (idx & 31) * 4;
            rb[h] = n < N ? __ldg(reinterpret_cast<const float4*>(B + (size_t)(k0 + kk) * N + n)) : make_float4(0.f, 0.f, 0.f, 0.f);
        }
    };
    auto store = [&](int buf) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int idx = tid + h * 256;
            if (!kWgrad) *reinterpret_cast<float4*>(&As[buf][(idx >> 2) * kAStr + (idx & 3) * 4]) = tf32x4(ra[h]);
            else         *reinterpret_cast<float4*>(&As[buf][(idx >> 5) * kBStr + (idx & 31) * 4]) = tf32x4(ra[h]);
            *reinterpret_cast<float4*>(&Bs[buf][(idx >> 5) * kBStr + (idx & 31) * 4]) = tf32x4(rb[h]);
        }
    };

    if (KT > 0) {
        load(0);
        store(0);
    }
    __syncthreads();
    for (int kt = 0; kt < KT; ++kt) {
        const int buf = kt & 1;
        if (kt + 1 < KT) load(kt + 1);
        const float* as = As[buf];
        const float* bs = Bs[buf];
#pragma unroll
        for (int ks = 0; ks < kBK; ks += 8) {
            uint32_t af[4][4], bf[4][2];
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const int r = wm * 64 + i * 16 + g;
                if (!kWgrad) {
                    af[i][0] = __float_as_uint(as[r * kAStr + ks + t4]);
                    af[i][1] = __float_as_uint(as[(r + 8) * kAStr + ks + t4]);
                    af[i][2] = __float_as_uint(as[r * kAStr + ks + t4 + 4]);
                    af[i][3] = __float_as_uint(as[(r + 8) * kAStr + ks + t4 + 4]);
                } else {
                    af[i][0] = __float_as_uint(as[(ks + t4) * kBStr + r]);
                    af[i][1] = __float_as_uint(as[(ks + t4) * kBStr + r + 8]);
                    af[i][2] = __float_as_uint(as[(ks + t4 + 4) * kBStr + r]);
                    af[i][3] = __float_as_uint(as[(ks + t4 + 4) * kBStr + r + 8]);
                }
            }
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const int c = wn * 32 + j * 8 + g;
                bf[j][0] = __float_as_uint(bs[(ks + t4) * kBStr + c]);
                bf[j][1] = __float_as_uint(bs[(ks + t4 + 4) * kBStr + c]);
            }
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) mma_tf32(acc[i][j], af[i], bf[j]);
        }
        if (kt + 1 < KT) store(buf ^ 1);
        __syncthreads();
    }

    float* o = kWgrad ? out + (size_t)blockIdx.z * Mrows * N : out;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
#pragma unroll
        for (int half = 0; half < 2; ++half) {
            const int m = m0 + wm * 64 + i * 16 + g + half * 8;
            if (m >= Mrows) continue;
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const int n = n0 + wn * 32 + j * 8 + 2 * t4;
                if (n >= N) continue;
                float2 v = make_float2(acc[i][j][2 * half], acc[i][j][2 * half + 1]);
                if (bias) { v.x += bias[n]; v.y += bias[n + 1]; }
                if (add) {
                    const float2 a = *reinterpret_cast<const float2*>(add + (size_t)m * N + n);
                    v.x += a.x; v.y += a.y;
                }
                *reinterpret_cast<float2*>(o + (size_t)m * N + n) = v;
            }
        }
    }
}

// dW[row][n] = sum over splits in order; conv0's padded rows (ci >= cin_real) are dropped.
__global__ void wgrad_reduce_kernel(const float* __restrict__ part, int splits, int cin_pad, int cin_real, int N,
                                    float* __restrict__ dw) {
    const size_t rows = (size_t)9 * cin_pad, total = rows * N;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const int r = (int)(i / N), n = (int)(i % N), tap = r / cin_pad, ci = r % cin_pad;
        if (ci >= cin_real) continue;
        float s = 0.f;
        for (int z = 0; z < splits; ++z) s += part[(size_t)z * total + i];
        dw[((size_t)tap * cin_real + ci) * N + n] = s;
    }
}

// ---- weight images ---------------------------------------------------------------------------------------------------
// conv0: W0p[tap][16][F] zero-padded from kernel[tap][2][F]
__global__ void pack_w0_kernel(const float* __restrict__ k, int F, float* __restrict__ w0p) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= 9 * kCin0 * F) return;
    const int n = i % F, ci = (i / F) % kCin0, tap = i / (F * kCin0);
    w0p[i] = ci < 2 ? k[((size_t)tap * 2 + ci) * F + n] : 0.f;
}

// input-gradient image: Wt[tap][co][ci] = W[8 - tap][ci][co]
__global__ void pack_wt_kernel(const float* __restrict__ w, int F, float* __restrict__ wt) {
    const size_t total = (size_t)9 * F * F;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const int ci = (int)(i % F), co = (int)((i / F) % F), tap = (int)(i / ((size_t)F * F));
        wt[i] = w[((size_t)(8 - tap) * F + ci) * F + co];
    }
}

// X0[b*64 + p][c] = planes[index[b]][c][p] for c < 2, 0 for the padding channels; an index outside [0, n_records)
// reads record 0 and raises *bad (the step then leaves the weights alone and reports NaN losses)
__global__ void gather_kernel(const uint8_t* __restrict__ planes, const int32_t* __restrict__ index, size_t n_records, int batch,
                              float* __restrict__ x0, int* __restrict__ bad) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= batch * 64 * kCin0) return;
    const int c = i % kCin0, m = i / kCin0, b = m >> 6, p = m & 63;
    int32_t r = index[b];
    if (r < 0 || (size_t)r >= n_records) {
        if (c == 0 && p == 0) *bad = 1;
        r = 0;
    }
    x0[i] = c < 2 ? (float)planes[(size_t)r * 128 + c * 64 + p] : 0.f;
}

// a group's copy of the batch's own records in batch order (the replicas receive these, not the dataset), with the
// substitution and *bad flag of gather_kernel: sp[b] = planes[index[b]], spol[b] = policy[index[b]], sz[b] = z[index[b]]
__global__ void stage_kernel(const uint8_t* __restrict__ planes, const float* __restrict__ policy, const float* __restrict__ z,
                             const int32_t* __restrict__ index, size_t n_records, int batch, uint8_t* __restrict__ sp,
                             float* __restrict__ spol, float* __restrict__ sz, int* __restrict__ bad) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= batch * 64) return;
    const int b = i >> 6, p = i & 63;
    int32_t r = index[b];
    if (r < 0 || (size_t)r >= n_records) {
        if (p == 0) *bad = 1;
        r = 0;
    }
    sp[(size_t)b * 128 + p] = planes[(size_t)r * 128 + p];
    sp[(size_t)b * 128 + 64 + p] = planes[(size_t)r * 128 + 64 + p];
    spol[(size_t)b * 64 + p] = policy[(size_t)r * 64 + p];
    if (p == 0) sz[b] = z[r];
}

// ---- BatchNormalization (training mode) ------------------------------------------------------------------------------
// Per-channel column reductions over the M = B*64 rows of a [M][ld] tensor (channels [0, C)): each CTA reduces 64 rows
// into partial[chunk][v][C] (threads over channels x row lanes, lanes combined in order); a finalize kernel adds the
// chunks in order.
enum RedMode { kSum = 0, kSqDev = 1, kBnGrad = 2, kHeadConvGrad = 3 };

template <int MODE>
__global__ void colred_partial_kernel(const float* __restrict__ y, const float* __restrict__ a, const float* __restrict__ gr,
                                      int ld, int ld2, int C, int M, const float* __restrict__ mean,
                                      const float* __restrict__ invstd, double* __restrict__ part) {
    constexpr int NV = MODE == kBnGrad ? 2 : MODE == kHeadConvGrad ? 3 : 1;
    __shared__ double sm[256 * NV];
    const int t = threadIdx.x, lanes = 256 / C, c = t % C, rl = t / C;
    const int r0 = blockIdx.x * kRowsPerChunk, r1 = min(r0 + kRowsPerChunk, M);
    double s[NV];
#pragma unroll
    for (int v = 0; v < NV; ++v) s[v] = 0.0;
    if (rl < lanes) {
        const float mu = (MODE == kSqDev || MODE == kBnGrad) ? mean[c] : 0.f;
        const float is = MODE == kBnGrad ? invstd[c] : 0.f;
        for (int m = r0 + rl; m < r1; m += lanes) {
            const float x = y[(size_t)m * ld + c];
            if (MODE == kSum) s[0] += x;
            if (MODE == kSqDev) { const double d = (double)x - mu; s[0] += d * d; }
            if (MODE == kBnGrad) {
                const float dz = a[(size_t)m * ld + c] > 0.f ? gr[(size_t)m * ld + c] : 0.f;
                s[0] += dz;
                s[1] += (double)dz * ((x - mu) * is);
            }
            if (MODE == kHeadConvGrad) {  // y = tower output [M][C], gr = head conv output gradient [M][ld2 = 3]
#pragma unroll
                for (int v = 0; v < 3; ++v) s[v] += (double)x * gr[(size_t)m * ld2 + v];
            }
        }
    }
#pragma unroll
    for (int v = 0; v < NV; ++v) sm[v * 256 + t] = s[v];
    __syncthreads();
    if (t < C) {
        for (int v = 0; v < NV; ++v) {
            double acc = 0.0;
            for (int l = 0; l < lanes; ++l) acc += sm[v * 256 + l * C + t];
            part[((size_t)blockIdx.x * NV + v) * C + t] = acc;
        }
    }
}

// Per-layer BN parameters and saved statistics.  off = blob offset of the conv kernel; the bias, gamma, beta, moving
// mean and moving variance follow at off + kf + {0, 1, 2, 3, 4} * C.
struct BnRef {
    size_t off, kf;
    int C;
};

template <int MODE>
__global__ void colred_finalize_kernel(const double* __restrict__ part, int chunks, int C, int M, BnRef bn,
                                       float* __restrict__ mean, float* __restrict__ invstd, float* __restrict__ sums,
                                       float* __restrict__ stat, float* __restrict__ grad) {
    constexpr int NV = MODE == kBnGrad ? 2 : MODE == kHeadConvGrad ? 3 : 1;
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= C) return;
    float s[NV];
    for (int v = 0; v < NV; ++v) {
        double acc = 0.0;
        for (int k = 0; k < chunks; ++k) acc += part[((size_t)k * NV + v) * C + c];
        s[v] = (float)(MODE <= kSqDev ? acc / M : acc);
    }
    const size_t base = bn.off + bn.kf;
    if (MODE == kSum) mean[c] = s[0];
    if (MODE == kSqDev) {
        const float var = s[0];  // biased, as used for normalisation
        invstd[c] = 1.f / sqrtf(var + kTrainBnEps);
        stat[base + 3 * bn.C + c] = mean[c];
        stat[base + 4 * bn.C + c] = var;
    }
    if (MODE == kBnGrad) {
        sums[c] = s[0];
        sums[C + c] = s[1];
        grad[base + 2 * bn.C + c] = s[0];  // beta
        grad[base + bn.C + c] = s[1];      // gamma
        grad[base + c] = 0.f;              // conv bias: exactly zero under training-mode BN (see DESIGN)
    }
    if (MODE == kHeadConvGrad) {
        // bn.off = policy_conv kernel [C][2], bn.kf = value_conv kernel offset [C][1]
        grad[bn.off + (size_t)c * 2] = s[0];
        grad[bn.off + (size_t)c * 2 + 1] = s[1];
        grad[bn.kf + c] = s[2];
    }
}

// A[m][c] = relu(gamma * (y - mean) * invstd + beta (+ res[m][c]))
__global__ void bn_apply_kernel(const float* __restrict__ y, const float* __restrict__ res, int ld, int C, int M,
                                const float* __restrict__ blob, BnRef bn, const float* __restrict__ mean,
                                const float* __restrict__ invstd, float* __restrict__ out) {
    const size_t total = (size_t)M * C;
    const float* gamma = blob + bn.off + bn.kf + bn.C;
    const float* beta = gamma + bn.C;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const int c = (int)(i % C);
        const size_t o = (i / C) * ld + c;
        float v = fmaf((y[o] - mean[c]) * invstd[c], gamma[c], beta[c]);
        if (res) v += res[o];
        out[o] = fmaxf(v, 0.f);
    }
}

// dy = gamma * invstd * (dz - (sum dz + xhat * sum dz*xhat) / M), dz = g where the layer's output is positive;
// dz_out (nullable) keeps dz for the skip connection of a residual block.  Visits M rows; M_norm is the batch's row count
// (M, except on a replica of a group, which holds a shard of the batch)
__global__ void bn_backward_kernel(const float* __restrict__ g, const float* __restrict__ a, const float* __restrict__ y, int ld,
                                   int C, int M, int M_norm, const float* __restrict__ blob, BnRef bn, const float* __restrict__ mean,
                                   const float* __restrict__ invstd, const float* __restrict__ sums, float* __restrict__ dy,
                                   float* __restrict__ dz_out) {
    const size_t total = (size_t)M * C;
    const float* gamma = blob + bn.off + bn.kf + bn.C;
    const float inv_m = 1.f / (float)M_norm;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const int c = (int)(i % C);
        const size_t o = (i / C) * ld + c;
        const float dz = a[o] > 0.f ? g[o] : 0.f;
        const float xh = (y[o] - mean[c]) * invstd[c];
        dy[o] = gamma[c] * invstd[c] * (dz - (sums[c] + xh * sums[C + c]) * inv_m);
        if (dz_out) dz_out[o] = dz;
    }
}

// ---- heads -----------------------------------------------------------------------------------------------------------
// 1x1 head convolutions: hc[m][0..1] = policy_conv, hc[m][2] = value_conv (+ biases); one warp per pixel.
__global__ void head_conv_kernel(const float* __restrict__ x, int F, int M, const float* __restrict__ blob, size_t off_pc,
                                 size_t off_vc, float* __restrict__ hc) {
    const int m = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (m >= M) return;
    double s0 = 0.0, s1 = 0.0, s2 = 0.0;
    for (int c = lane; c < F; c += 32) {
        const double v = x[(size_t)m * F + c];
        s0 += v * blob[off_pc + 2 * c];
        s1 += v * blob[off_pc + 2 * c + 1];
        s2 += v * blob[off_vc + c];
    }
    for (int o = 16; o; o >>= 1) {
        s0 += __shfl_xor_sync(0xffffffffu, s0, o);
        s1 += __shfl_xor_sync(0xffffffffu, s1, o);
        s2 += __shfl_xor_sync(0xffffffffu, s2, o);
    }
    if (lane == 0) {
        hc[(size_t)m * 3] = (float)(s0 + blob[off_pc + 2 * F]);
        hc[(size_t)m * 3 + 1] = (float)(s1 + blob[off_pc + 2 * F + 1]);
        hc[(size_t)m * 3 + 2] = (float)(s2 + blob[off_vc + F]);
    }
}

struct HeadOffs {
    size_t pfk, pfb, v1k, v1b, v2k, v2b;
};

// Per record: Dense(128->64) + softmax + policy loss, Dense(64->V, relu) + Dense(V->1, tanh) + value loss, and their
// backward down to the gradient of the head BN+ReLU outputs (dh[m][3], before the ReLU mask).  One CTA per record.
// Computed in fp64 (a few thousand operations per record): 1 - v^2 next to |v| = 1 and the softmax / log loss lose
// most of fp32's digits to cancellation.
__global__ void __launch_bounds__(256) head_fc_kernel(const float* __restrict__ ah, const float* __restrict__ blob, HeadOffs o, int V,
                                                      const float* __restrict__ policy, const float* __restrict__ z,
                                                      const int32_t* __restrict__ index, size_t n_records, int batch,
                                                      float* __restrict__ hp_out, float* __restrict__ hv_out, float* __restrict__ dl_out,
                                                      float* __restrict__ h1_out, float* __restrict__ dh1_out, float* __restrict__ dv_out,
                                                      float* __restrict__ loss_p, float* __restrict__ loss_v, float* __restrict__ dh) {
    extern __shared__ double shd[];
    double* hp = shd;         // [128] = c * 64 + p (channels_first flatten)
    double* hv = hp + 128;    // [64]
    double* lg = hv + 64;     // [64] logits, then probabilities
    double* gg = lg + 64;     // [64] d loss / d p
    double* dl = gg + 64;     // [64] d loss / d logits
    double* red = dl + 64;    // [8] scalars
    double* h1 = red + 8;     // [V]
    double* dh1 = h1 + V;     // [V]
    const int t = threadIdx.x, b = blockIdx.x;
    const double inv_b = 1.0 / (double)batch;
    int32_t r = index[b];
    if (r < 0 || (size_t)r >= n_records) r = 0;
    const float* y = policy + (size_t)r * 64;
    const size_t mb = (size_t)b * 64;
    if (t < 192) {
        const int c = t >> 6, p = t & 63;
        const double v = ah[(mb + p) * 3 + c];
        if (c < 2) hp[c * 64 + p] = v; else hv[p] = v;
    }
    __syncthreads();
    if (t < 64) {
        double acc = blob[o.pfb + t];
        for (int i = 0; i < 128; ++i) acc += hp[i] * blob[o.pfk + i * 64 + t];
        lg[t] = acc;
    }
    for (int j = t; j < V; j += 256) {
        double acc = blob[o.v1b + j];
        for (int i = 0; i < 64; ++i) acc += hv[i] * blob[o.v1k + (size_t)i * V + j];
        h1[j] = acc > 0.0 ? acc : 0.0;
    }
    __syncthreads();
    if (t == 0) {
        double mx = -INFINITY;
        for (int i = 0; i < 64; ++i) mx = fmax(mx, lg[i]);
        double s = 0.0;
        for (int i = 0; i < 64; ++i) s += exp(lg[i] - mx);
        red[0] = mx;
        red[1] = s;
    }
    if (t == 32) {
        double acc = blob[o.v2b];
        for (int j = 0; j < V; ++j) acc += h1[j] * blob[o.v2k + j];
        red[2] = tanh(acc);
    }
    __syncthreads();
    if (t < 64) {
        const double p = exp(lg[t] - red[0]) / red[1];
        lg[t] = p;
        gg[t] = -(double)y[t] / (p + (double)kLogEps);
    }
    __syncthreads();
    if (t == 0) {
        double lp = 0.0, pg = 0.0;
        for (int i = 0; i < 64; ++i) {
            lp -= (double)y[i] * log(lg[i] + (double)kLogEps);
            pg += lg[i] * gg[i];
        }
        const double v = red[2], d = v - (double)z[r];
        loss_p[b] = (float)lp;
        loss_v[b] = (float)(d * d);
        red[3] = pg;
        red[4] = 2.0 * d * (1.0 - v * v) * inv_b;  // d loss / d value pre-activation
        dv_out[b] = (float)red[4];
    }
    __syncthreads();
    if (t < 64) {
        dl[t] = lg[t] * (gg[t] - red[3]) * inv_b;
        dl_out[(size_t)b * 64 + t] = (float)dl[t];
    }
    for (int j = t; j < V; j += 256) {
        dh1[j] = h1[j] > 0.0 ? red[4] * blob[o.v2k + j] : 0.0;
        h1_out[(size_t)b * V + j] = (float)h1[j];
        dh1_out[(size_t)b * V + j] = (float)dh1[j];
    }
    __syncthreads();
    if (t < 128) {
        hp_out[(size_t)b * 128 + t] = (float)hp[t];
        double acc = 0.0;
        for (int j = 0; j < 64; ++j) acc += dl[j] * blob[o.pfk + t * 64 + j];
        dh[(mb + (t & 63)) * 3 + (t >> 6)] = (float)acc;
    } else if (t < 192) {
        const int i = t - 128;
        hv_out[(size_t)b * 64 + i] = (float)hv[i];
        double acc = 0.0;
        for (int j = 0; j < V; ++j) acc += dh1[j] * blob[o.v1k + (size_t)i * V + j];
        dh[(mb + i) * 3 + 2] = (float)acc;
    }
}

// Dense-layer gradients summed over the batch in record order, and the batch-mean policy / value losses.
__global__ void head_fc_grad_kernel(const float* __restrict__ hp, const float* __restrict__ hv, const float* __restrict__ dl,
                                    const float* __restrict__ h1, const float* __restrict__ dh1, const float* __restrict__ dv,
                                    const float* __restrict__ loss_p, const float* __restrict__ loss_v, int V, int batch, HeadOffs o,
                                    float* __restrict__ grad, float* __restrict__ loss_pv) {
    const int n_pfk = 128 * 64, n_pfb = 64, n_v1k = 64 * V, n_v1b = V, n_v2k = V;
    const int total = n_pfk + n_pfb + n_v1k + n_v1b + n_v2k + 1 + 1;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    double s = 0.0;  // sums over the batch cancel across records: accumulate in fp64
    int k = i;
    if (k < n_pfk) {
        const int a = k / 64, j = k % 64;
        for (int b = 0; b < batch; ++b) s += (double)hp[(size_t)b * 128 + a] * dl[(size_t)b * 64 + j];
        grad[o.pfk + k] = (float)s;
        return;
    }
    k -= n_pfk;
    if (k < n_pfb) {
        for (int b = 0; b < batch; ++b) s += dl[(size_t)b * 64 + k];
        grad[o.pfb + k] = (float)s;
        return;
    }
    k -= n_pfb;
    if (k < n_v1k) {
        const int a = k / V, j = k % V;
        for (int b = 0; b < batch; ++b) s += (double)hv[(size_t)b * 64 + a] * dh1[(size_t)b * V + j];
        grad[o.v1k + k] = (float)s;
        return;
    }
    k -= n_v1k;
    if (k < n_v1b) {
        for (int b = 0; b < batch; ++b) s += dh1[(size_t)b * V + k];
        grad[o.v1b + k] = (float)s;
        return;
    }
    k -= n_v1b;
    if (k < n_v2k) {
        for (int b = 0; b < batch; ++b) s += (double)h1[(size_t)b * V + k] * dv[b];
        grad[o.v2k + k] = (float)s;
        return;
    }
    k -= n_v2k;
    if (k == 0) {
        for (int b = 0; b < batch; ++b) s += dv[b];
        grad[o.v2b] = (float)s;
        return;
    }
    float lp = 0.f, lv = 0.f;
    for (int b = 0; b < batch; ++b) { lp += loss_p[b]; lv += loss_v[b]; }
    loss_pv[0] = lp / (float)batch;
    loss_pv[1] = lv / (float)batch;
}

// gradient of the tower output from the head convolutions: g[m][c] = sum_h dyh[m][h] * W_h[c]
__global__ void head_conv_dgrad_kernel(const float* __restrict__ dyh, const float* __restrict__ blob, size_t off_pc, size_t off_vc,
                                       int F, int M, float* __restrict__ g) {
    const size_t total = (size_t)M * F;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const int c = (int)(i % F);
        const size_t m = i / F;
        g[i] = dyh[m * 3] * blob[off_pc + 2 * c] + dyh[m * 3 + 1] * blob[off_pc + 2 * c + 1] + dyh[m * 3 + 2] * blob[off_vc + c];
    }
}

// ---- update ----------------------------------------------------------------------------------------------------------
// Keras SGD with momentum: v = mu * v - lr * g; w = w + v, with g += 2 * l2 * w for kernels (kernel_regularizer);
// moving statistics: w = bn_mom * w + (1 - bn_mom) * batch statistic.  Also the L2 sum of the pre-update kernels.
__global__ void __launch_bounds__(256) update_kernel(float* __restrict__ w, float* __restrict__ vel, float* __restrict__ grad,
                                                     const float* __restrict__ stat, const uint8_t* __restrict__ kind, size_t n,
                                                     float lr, float mu, float l2, float bn_mom, const int* __restrict__ bad,
                                                     float* __restrict__ l2_part) {
    __shared__ float sm[256];
    const bool skip = *bad != 0;
    float s = 0.f;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const uint8_t k = kind[i];
        const float x = w[i];
        if (k == kKernel) s = fmaf(x, x, s);
        if (skip) continue;
        if (k <= kTrainable) {
            const float gi = k == kKernel ? fmaf(2.f * l2, x, grad[i]) : grad[i];
            grad[i] = gi;
            const float v = mu * vel[i] - lr * gi;
            vel[i] = v;
            w[i] = x + v;
        } else {
            grad[i] = 0.f;
            w[i] = bn_mom * x + (1.f - bn_mom) * stat[i];
        }
    }
    sm[threadIdx.x] = s;
    __syncthreads();
    for (int o = 128; o; o >>= 1) {
        if (threadIdx.x < o) sm[threadIdx.x] += sm[threadIdx.x + o];
        __syncthreads();
    }
    if (threadIdx.x == 0) l2_part[blockIdx.x] = sm[0];
}

__global__ void loss_kernel(const float* __restrict__ l2_part, const float* __restrict__ loss_pv, float l2, const int* __restrict__ bad,
                            float* __restrict__ loss) {
    if (threadIdx.x) return;
    float s = 0.f;
    for (int i = 0; i < kUpdateBlocks; ++i) s += l2_part[i];
    if (*bad) {
        loss[0] = loss[1] = loss[2] = NAN;
        return;
    }
    loss[0] = loss_pv[0] + loss_pv[1] + l2 * s;
    loss[1] = loss_pv[0];
    loss[2] = loss_pv[1];
}

__global__ void mask_grad_kernel(const float* __restrict__ grad, const uint8_t* __restrict__ kind, size_t n, float* __restrict__ out) {
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
        out[i] = kind[i] <= kTrainable ? grad[i] : 0.f;
}

// dynamic shared memory of head_fc_kernel
inline size_t head_fc_smem(int V) { return (size_t)(128 + 64 * 4 + 8 + 2 * V) * sizeof(double); }

inline int chunks_of(int M) { return (M + kRowsPerChunk - 1) / kRowsPerChunk; }

inline unsigned grid_for(size_t n, int threads = 256, size_t cap = 4096) {
    size_t b = (n + threads - 1) / threads;
    return (unsigned)(b < 1 ? 1 : b > cap ? cap : b);
}

}  // namespace
}  // namespace rz

using namespace rz;

struct rz_trainer {
    rz_net_cfg net;
    rz_train_cfg cfg;
    int device;
    bool loaded;
    int F, R, V, L;  // L = 1 + 2R tower convolutions
    size_t n;        // blob floats
    size_t off_pc, off_vc;  // policy / value head conv kernels
    HeadOffs ho;
    std::vector<size_t> conv_off;  // kernel offset of tower convolution l

    float *blob, *vel, *grad, *stat;
    uint8_t* kind;
    float *x0, *w0p, *wt;         // input planes [M][16]; conv0 weight image; input-gradient images [2R][9F*F]
    float *y, *a;                 // [L][M][F] conv outputs (pre-BN) and layer outputs
    float *g, *g1, *dy, *dz;      // [M][F] backward buffers
    float *hc, *ah, *dh, *dyh;    // [M][3] head conv outputs, head BN+ReLU outputs, their gradients
    float *hp, *hv, *dl, *h1, *dh1, *dv, *lp, *lv;  // per-record head tensors
    float *stats;                 // [L + 2][4][F]: mean, invstd, sum dz, sum dz*xhat
    double *part;                 // column-reduction partials [max_batch][3][F] ([act][3][F] on replicas 1..)
    float *wpart;                 // weight-gradient split-K partials [wslot]
    size_t wslot;                 // floats of the split partials of the largest layer at max_batch
    float *l2_part, *loss_pv;
    int* bad;
    size_t act;                   // records the activation and backward buffers hold (max_batch for a single trainer)

    // The handle is replica 0, the primary, of a data-parallel group (rz_trainer_create_group).  A single trainer is the
    // group of that one replica and owns nothing below `reps`.
    std::vector<rz_trainer*> reps;  // every replica, reps[0] = this
    cudaStream_t stream;          // replicas 1..: the stream the trainer owns (the primary runs on the caller's stream)
    cudaEvent_t ev;               // marks this replica's progress at each exchange
    uint8_t* sp;                  // staged batch records: planes [.][128], policy [.][64], z [.] (primary: max_batch)
    float *spol, *sz;
    int32_t* iota;                // replicas 1..: identity index [act]: the staged records are the replica's dataset
    float* wgather;               // primary: every layer's weight-gradient split partials [L][wslot], reduced after the join

    // test hooks of a single trainer (rz_trainer_debug_tensor_dev, rz_trainer_debug_keep_backward)
    int last_batch;               // batch of the last step; 0 before the first
    float* taps;                  // [L][3][64 * act][F]: each tower layer's G (gradient of A), dY and dz; null when off
    bool taps_valid;              // the last step ran with the taps on
};

namespace {

void trainer_free(rz_trainer* t) {
    float* bufs[] = {t->blob, t->vel, t->grad, t->stat, t->x0, t->w0p, t->wt, t->y, t->a, t->g, t->g1, t->dy, t->dz, t->hc, t->ah,
                     t->dh, t->dyh, t->hp, t->hv, t->dl, t->h1, t->dh1, t->dv, t->lp, t->lv, t->stats, t->wpart,
                     t->l2_part, t->loss_pv, t->spol, t->sz, t->wgather, t->taps};
    for (float* p : bufs) cudaFree(p);
    cudaFree(t->part);
    cudaFree(t->kind);
    cudaFree(t->bad);
    cudaFree(t->sp);
    cudaFree(t->iota);
    if (t->stream) cudaStreamDestroy(t->stream);
    if (t->ev) cudaEventDestroy(t->ev);
}

int wgrad_splits(int cin, int F, int batch) {
    const int tiles = ((9 * cin + kBM - 1) / kBM) * ((F + kBN - 1) / kBN);
    int s = (kWgradTargetBlocks + tiles - 1) / tiles;
    return s < batch ? s : batch;
}

// records per weight-gradient split of a convolution with cin input channels (launch_wgrad)
int wgrad_per(int cin, int F, int batch) {
    const int splits = wgrad_splits(cin, F, batch);
    return (batch + splits - 1) / splits;
}

// Shards of a step: replica r trains on records [bounds[r], bounds[r + 1]).  The boundaries sit on the weight-gradient
// split grid of the F->F convolutions (conv0's grid without residual blocks), so every split of those layers lies
// inside one shard; the grid's cells are dealt out as evenly as possible, the larger shares first.
void shard_plan(int F, int R, int batch, int n, int* bounds) {
    const int per = wgrad_per(R ? F : kCin0, F, batch), cells = (batch + per - 1) / per;
    const int q = cells / n, rem = cells % n;
    for (int r = 0; r <= n; ++r) bounds[r] = std::min(batch, per * (r * q + std::min(r, rem)));
}

// conv0's weight-gradient splits are finer than the tower's and may straddle the end of a shard: a replica computes the
// splits that start in its shard, which takes the first `ov` records of the next shard as well
struct Conv0Share {
    int z0, nz;         // its conv0 splits [z0, z0 + nz)
    int row0, rows;     // the records they cover, relative to the shard's first
    int ov;             // records past the end of the shard (rows of the next replica)
};

Conv0Share conv0_share(int F, int batch, int b0, int n) {
    if (n == 0) return Conv0Share{0, 0, 0, 0, 0};
    const int per0 = wgrad_per(kCin0, F, batch), e = b0 + n;
    const int z0 = (b0 + per0 - 1) / per0, z1 = (e + per0 - 1) / per0;
    const int end = std::min(z1 * per0, batch);
    return z1 > z0 ? Conv0Share{z0, z1 - z0, z0 * per0 - b0, end - z0 * per0, end - e} : Conv0Share{z0, 0, 0, 0, 0};
}

int launch_conv(const float* in, int cin, const float* w, int F, const float* bias, const float* add, float* out, int M,
                cudaStream_t st) {
    dim3 grid((M + kBM - 1) / kBM, (F + kBN - 1) / kBN);
    conv_gemm_tf32_kernel<false><<<grid, 256, 0, st>>>(in, cin, w, F, bias, add, out, M, 0);
    RZ_LAUNCH_CHECK();
    return RZ_OK;
}

// `nz` consecutive split-K partials of a convolution's weight gradient into part[nz][9 * cin][F]: the k-th covers records
// [k * per, (k + 1) * per) of the input `in` [rows * 64][cin] and of the output gradient dyp [rows * 64][F].  Given dw,
// they are all of the layer's splits and are reduced at once into dw (blob layout [9][cin_real][F]).
int launch_wgrad(const float* in, int cin, int cin_real, const float* dyp, int F, int rows, int nz, int per, float* part, float* dw,
                 cudaStream_t st) {
    dim3 grid((9 * cin + kBM - 1) / kBM, (F + kBN - 1) / kBN, nz);
    conv_gemm_tf32_kernel<true><<<grid, 256, 0, st>>>(in, cin, dyp, F, nullptr, nullptr, part, rows * 64, per * 64);
    if (dw) wgrad_reduce_kernel<<<grid_for((size_t)9 * cin * F), 256, 0, st>>>(part, nz, cin, cin_real, F, dw);
    RZ_LAUNCH_CHECK();
    return RZ_OK;
}

// A tensor of the step that every replica holds, named once for all of them: p->*buf + layer * (p's layer stride) + col
using TrainerBuf = float* rz_trainer::*;
struct Operand {
    TrainerBuf buf = nullptr;  // null: no operand
    int layer = 0, col = 0;
};

// The dataset a replica reads its shard from
struct Records {
    const uint8_t* planes;
    const float *policy, *z;
    const int32_t* index;
    size_t n;
};

// ---- the training step -----------------------------------------------------------------------------------------------
// One schedule for a single trainer and for a data-parallel group.  The batch is split into the shards of shard_plan, one
// per replica, and every sum over the batch is taken by the same operations in the same order whatever the split:
//  * column reductions (BN statistics, BN and head-conv gradients): every replica writes the per-record partials of its
//    shard; the primary gathers them into its `part` in batch order and runs the finalize over all chunks with the global
//    M; the replicas copy back the finalized mean / invstd / sums (and the batch statistics of the moving averages);
//  * dense heads: the per-record head tensors are gathered on the primary, which runs head_fc_grad_kernel on the batch;
//  * weight gradients: every replica computes the split-K partials of its own splits (conv0's straddling split with the
//    next replica's first rows); the primary gathers them into one slot per layer and reduces every layer in split order;
//  * the primary then hands its whole gradient and the `bad` flag to every replica, and every replica runs update_kernel
//    on them, so weights, momentum and moving statistics stay identical without a weight broadcast.
// Transport is cudaMemcpyPeerAsync (a device-to-device copy between replicas on one device) ordered by one event per
// replica.  At every exchange the primary waits on every replica (empty ones included), and the exchange ends with every
// replica waiting on the primary, so no buffer a copy reads is rewritten before the copy has run; the replicas join the
// caller's stream at the end and wait on it at the start.  A replica with an empty shard launches nothing but its copy
// of the moving-average statistics, the gradient copy and update_kernel.
// The primary's shard starts the batch, so it reads the caller's dataset through the caller's index; replicas 1.. read
// records the primary staged for them.  A single trainer is the group of one replica: its shard is the batch, every
// exchange is a loop over no replica, and it enqueues no staging, event or copy.  Its weight-gradient partials need no
// slot either: each layer's go to `wpart` and are reduced at once.
int step(rz_trainer* t, const uint8_t* planes, const float* policy, const float* z, const int32_t* index, size_t n_records, int batch,
         float lr, float* loss, cudaStream_t st) {
    const int F = t->F, R = t->R, L = t->L, V = t->V, n = (int)t->reps.size(), Mg = batch * 64;
    int bounds[65];
    shard_plan(F, R, batch, n, bounds);
    const int per = wgrad_per(R ? F : kCin0, F, batch), per0 = wgrad_per(kCin0, F, batch);
    auto on = [&](int r) { return n > 1 ? cudaSetDevice(t->reps[r]->device) : cudaSuccess; };  // alone, t's device is current
    auto S = [&](int r) { return r ? t->reps[r]->stream : st; };
    auto b0 = [&](int r) { return bounds[r]; };
    auto nr = [&](int r) { return bounds[r + 1] - bounds[r]; };
    auto records = [&](int r) {
        const rz_trainer* p = t->reps[r];
        return r ? Records{p->sp, p->spol, p->sz, p->iota, p->act} : Records{planes, policy, z, index, n_records};
    };
    auto at = [&](rz_trainer* p, Operand o) { return o.buf ? p->*o.buf + (size_t)o.layer * 64 * p->act * F + o.col : nullptr; };
    auto Y = [](int l) { return Operand{&rz_trainer::y, l}; };
    auto A = [](int l) { return Operand{&rz_trainer::a, l}; };
    const Operand none{}, g{&rz_trainer::g}, g1{&rz_trainer::g1}, dy{&rz_trainer::dy}, dz{&rz_trainer::dz};
    const Operand hc{&rz_trainer::hc}, ah{&rz_trainer::ah}, dh{&rz_trainer::dh}, dyh{&rz_trainer::dyh};
    auto value = [](Operand o) { return Operand{o.buf, 0, 2}; };  // the value head's column of a [M][3] head tensor
    auto ST = [&](rz_trainer* p, int l) { return p->stats + (size_t)l * 4 * F; };
    auto bnref = [&](int l) { return BnRef{t->conv_off[l], (size_t)9 * (l ? F : 2) * F, F}; };
    auto peer = [&](void* dst, int r_dst, const void* src, int r_src, size_t bytes, cudaStream_t s) {
        return bytes ? cudaMemcpyPeerAsync(dst, t->reps[r_dst]->device, src, t->reps[r_src]->device, bytes, s) : cudaSuccess;
    };
    const int chunks = batch;  // kRowsPerChunk = 64 rows: one column-reduction partial per record
    // the capacities the trainer was created with: a shard and its conv0 overflow fit the replica's buffers, and every
    // layer's split partials fit `wpart` and one gradient slot
    for (int r = 0; r < n; ++r)
        RZ_REQUIRE((size_t)nr(r) + conv0_share(F, batch, b0(r), nr(r)).ov <= t->reps[r]->act,
                   "training step: shard of replica %d exceeds its buffers", r);
    RZ_REQUIRE((size_t)((batch + per - 1) / per) * 9 * (R ? F : kCin0) * F <= t->wslot &&
                   (size_t)((batch + per0 - 1) / per0) * 9 * kCin0 * F <= t->wslot,
               "training step: weight-gradient splits exceed their scratch");
    t->last_batch = batch;
    t->taps_valid = t->taps != nullptr;

    // the primary stages the batch for replicas 1.., which copy their shard (and conv0's overflow records); every
    // replica expands its x0
    RZ_CUDA_TRY(cudaMemsetAsync(t->bad, 0, sizeof(int), st));
    if (n > 1) {
        stage_kernel<<<(Mg + 255) / 256, 256, 0, st>>>(planes, policy, z, index, n_records, batch, t->sp, t->spol, t->sz, t->bad);
        RZ_LAUNCH_CHECK();
        RZ_CUDA_TRY(cudaEventRecord(t->ev, st));
    }
    for (int r = 0; r < n; ++r) {
        rz_trainer* p = t->reps[r];
        const cudaStream_t s = S(r);
        RZ_CUDA_TRY(on(r));
        const int rows = nr(r) + (R ? conv0_share(F, batch, b0(r), nr(r)).ov : 0);
        if (r) {
            RZ_CUDA_TRY(cudaStreamWaitEvent(s, t->ev, 0));
            RZ_CUDA_TRY(peer(p->sp, r, t->sp + (size_t)b0(r) * 128, 0, (size_t)rows * 128, s));
            RZ_CUDA_TRY(peer(p->spol, r, t->spol + (size_t)b0(r) * 64, 0, (size_t)rows * 64 * sizeof(float), s));
            RZ_CUDA_TRY(peer(p->sz, r, t->sz + b0(r), 0, (size_t)rows * sizeof(float), s));
        }
        if (!nr(r)) continue;
        const Records rec = records(r);
        gather_kernel<<<(rows * 64 * kCin0 + 255) / 256, 256, 0, s>>>(rec.planes, rec.index, rec.n, rows, p->x0, p->bad);
        pack_w0_kernel<<<(9 * kCin0 * F + 255) / 256, 256, 0, s>>>(p->blob + t->conv_off[0], F, p->w0p);
        for (int l = 1; l < L; ++l)
            pack_wt_kernel<<<grid_for((size_t)9 * F * F), 256, 0, s>>>(p->blob + t->conv_off[l], F, p->wt + (size_t)(l - 1) * 9 * F * F);
        RZ_LAUNCH_CHECK();
    }

    // the replicas' partials of `rec` doubles per record go to the primary's `part` in batch order
    auto gather_part = [&](size_t rec) -> int {
        for (int r = 1; r < n; ++r) {
            RZ_CUDA_TRY(on(r));
            RZ_CUDA_TRY(cudaEventRecord(t->reps[r]->ev, S(r)));
        }
        RZ_CUDA_TRY(on(0));
        for (int r = 1; r < n; ++r) {
            RZ_CUDA_TRY(cudaStreamWaitEvent(st, t->reps[r]->ev, 0));
            if (!nr(r)) continue;
            RZ_CUDA_TRY(peer(t->part + (size_t)b0(r) * rec, 0, t->reps[r]->part, r, (size_t)nr(r) * rec * sizeof(double), st));
        }
        return RZ_OK;
    };
    // after the primary's finalize: the replicas wait for it and copy layer l's finalized statistics (those with an empty
    // shard never read them) and the `stat_n` moving-average batch statistics at stat_off (which update_kernel reads)
    auto release = [&](int l, size_t stat_off, size_t stat_n) -> int {
        if (n == 1) return RZ_OK;
        RZ_CUDA_TRY(on(0));
        RZ_CUDA_TRY(cudaEventRecord(t->ev, st));
        for (int r = 1; r < n; ++r) {
            rz_trainer* p = t->reps[r];
            RZ_CUDA_TRY(on(r));
            RZ_CUDA_TRY(cudaStreamWaitEvent(p->stream, t->ev, 0));
            if (l >= 0 && nr(r)) RZ_CUDA_TRY(peer(ST(p, l), r, ST(t, l), 0, (size_t)4 * F * sizeof(float), p->stream));
            RZ_CUDA_TRY(peer(p->stat + stat_off, r, t->stat + stat_off, 0, stat_n * sizeof(float), p->stream));
        }
        return RZ_OK;
    };
    // launch(r, replica, rows, stream) on every replica with a non-empty shard
    auto partial_each = [&](auto launch) -> int {
        for (int r = 0; r < n; ++r) {
            if (!nr(r)) continue;
            RZ_CUDA_TRY(on(r));
            if constexpr (std::is_void_v<decltype(launch(r, t, 0, st))>) launch(r, t->reps[r], nr(r) * 64, S(r));
            else RZ_TRY(launch(r, t->reps[r], nr(r) * 64, S(r)));
            RZ_LAUNCH_CHECK();
        }
        return RZ_OK;
    };
    // training-mode BN forward of layer slot l over channels [0, C) of yp [rows][ld]: statistics, then normalise
    // (+ residual `res`) + ReLU into out
    auto bn_forward = [&](Operand yp, Operand res, int ld, int C, BnRef bn, int l, Operand out) -> int {
        RZ_TRY(partial_each([&](int, rz_trainer* p, int M, cudaStream_t s) {
            colred_partial_kernel<kSum><<<chunks_of(M), 256, 0, s>>>(at(p, yp), nullptr, nullptr, ld, 0, C, M, nullptr, nullptr, p->part);
        }));
        RZ_TRY(gather_part(C));
        colred_finalize_kernel<kSum><<<1, 256, 0, st>>>(t->part, chunks, C, Mg, bn, ST(t, l), ST(t, l) + F, nullptr, t->stat, t->grad);
        RZ_LAUNCH_CHECK();
        RZ_TRY(release(l, 0, 0));
        RZ_TRY(partial_each([&](int, rz_trainer* p, int M, cudaStream_t s) {
            colred_partial_kernel<kSqDev><<<chunks_of(M), 256, 0, s>>>(at(p, yp), nullptr, nullptr, ld, 0, C, M, ST(p, l), nullptr, p->part);
        }));
        RZ_TRY(gather_part(C));
        colred_finalize_kernel<kSqDev><<<1, 256, 0, st>>>(t->part, chunks, C, Mg, bn, ST(t, l), ST(t, l) + F, nullptr, t->stat, t->grad);
        RZ_LAUNCH_CHECK();
        RZ_TRY(release(l, bn.off + bn.kf + 3 * (size_t)bn.C, 2 * (size_t)bn.C));
        return partial_each([&](int, rz_trainer* p, int M, cudaStream_t s) {
            bn_apply_kernel<<<grid_for((size_t)M * C), 256, 0, s>>>(at(p, yp), at(p, res), ld, C, M, p->blob, bn, ST(p, l), ST(p, l) + F,
                                                                  at(p, out));
        });
    };
    // BN + ReLU backward of layer slot l: gp = gradient of the layer output ap; writes dyp (gradient of the conv output yp)
    // and, when dz_out is given, the gradient below the ReLU (what the skip connection carries); the gamma / beta
    // gradients go into the primary's grad
    auto bn_backward = [&](Operand gp, Operand ap, Operand yp, int ld, int C, BnRef bn, int l, Operand dyp, Operand dz_out) -> int {
        RZ_TRY(partial_each([&](int, rz_trainer* p, int M, cudaStream_t s) {
            colred_partial_kernel<kBnGrad><<<chunks_of(M), 256, 0, s>>>(at(p, yp), at(p, ap), at(p, gp), ld, 0, C, M, ST(p, l), ST(p, l) + F,
                                                                      p->part);
        }));
        RZ_TRY(gather_part(2 * (size_t)C));
        colred_finalize_kernel<kBnGrad><<<1, 256, 0, st>>>(t->part, chunks, C, Mg, bn, ST(t, l), ST(t, l) + F, ST(t, l) + 2 * F, t->stat,
                                                           t->grad);
        RZ_LAUNCH_CHECK();
        RZ_TRY(release(l, 0, 0));
        RZ_TRY(partial_each([&](int, rz_trainer* p, int M, cudaStream_t s) {
            bn_backward_kernel<<<grid_for((size_t)M * C), 256, 0, s>>>(at(p, gp), at(p, ap), at(p, yp), ld, C, M, Mg, p->blob, bn, ST(p, l),
                                                                     ST(p, l) + F, ST(p, l) + 2 * F, at(p, dyp), at(p, dz_out));
        }));
        if (t->taps && l < L) {  // test hook, single trainers only: keep this tower layer's G, dY and dz before they are reused
            const size_t bytes = (size_t)Mg * F * sizeof(float), stride = (size_t)64 * t->act * F;
            float* tap = t->taps + (size_t)l * 3 * stride;
            RZ_CUDA_TRY(cudaMemcpyAsync(tap, at(t, gp), bytes, cudaMemcpyDeviceToDevice, st));
            RZ_CUDA_TRY(cudaMemcpyAsync(tap + stride, at(t, dyp), bytes, cudaMemcpyDeviceToDevice, st));
            if (dz_out.buf) RZ_CUDA_TRY(cudaMemcpyAsync(tap + 2 * stride, at(t, dz_out), bytes, cudaMemcpyDeviceToDevice, st));
        }
        return RZ_OK;
    };
    // split partials [z0, z0 + nz) of layer l's weight gradient, computed by replica r from its rows `in` and `dyp`.  A
    // single replica reduces them at once from its wpart.  In a group the primary writes into the layer's slot and a
    // replica into its wpart and on, and every layer is reduced after the join.
    auto wgrad = [&](int l, int r, const float* in, const float* dyp, int rows, int z0, int nz) -> int {
        if (!nz) return RZ_OK;
        rz_trainer* p = t->reps[r];
        const int cin = l ? F : kCin0;
        const size_t slice = (size_t)9 * cin * F;
        float* slot = n > 1 ? t->wgather + (size_t)l * t->wslot + (size_t)z0 * slice : nullptr;
        RZ_TRY(launch_wgrad(in, cin, l ? F : 2, dyp, F, rows, nz, l ? per : per0, slot && !r ? slot : p->wpart,
                            slot ? nullptr : t->grad + t->conv_off[l], S(r)));
        if (r) RZ_CUDA_TRY(peer(slot, 0, p->wpart, r, (size_t)nz * slice * sizeof(float), S(r)));
        return RZ_OK;
    };

    // forward
    for (int l = 0; l < L; ++l) {
        RZ_TRY(partial_each([&](int, rz_trainer* p, int M, cudaStream_t s) {
            const float* in = l ? at(p, A(l - 1)) : p->x0;
            const float* w = l ? p->blob + t->conv_off[l] : p->w0p;
            return launch_conv(in, l ? F : kCin0, w, F, p->blob + t->conv_off[l] + bnref(l).kf, nullptr, at(p, Y(l)), M, s);
        }));
        const Operand res = (l >= 2 && l % 2 == 0) ? A(l - 2) : none;  // conv2 of a block adds the block input
        RZ_TRY(bn_forward(Y(l), res, F, F, bnref(l), l, A(l)));
    }
    const Operand tower = A(L - 1);
    RZ_TRY(partial_each([&](int, rz_trainer* p, int M, cudaStream_t s) {
        head_conv_kernel<<<(M * 32 + 255) / 256, 256, 0, s>>>(at(p, tower), F, M, p->blob, t->off_pc, t->off_vc, p->hc);
    }));
    const BnRef bpc{t->off_pc, (size_t)F * 2, 2}, bvc{t->off_vc, (size_t)F, 1};
    RZ_TRY(bn_forward(hc, none, 3, 2, bpc, L, ah));
    RZ_TRY(bn_forward(value(hc), none, 3, 1, bvc, L + 1, value(ah)));

    // loss and head backward; the per-record head tensors go to the primary
    const size_t fc_smem = head_fc_smem(V);
    RZ_TRY(partial_each([&](int r, rz_trainer* p, int M, cudaStream_t s) {
        const Records rec = records(r);
        head_fc_kernel<<<M / 64, 256, fc_smem, s>>>(p->ah, p->blob, t->ho, V, rec.policy, rec.z, rec.index, rec.n, batch, p->hp, p->hv,
                                                    p->dl, p->h1, p->dh1, p->dv, p->lp, p->lv, p->dh);
    }));
    for (int r = 1; r < n; ++r) {
        RZ_CUDA_TRY(on(r));
        RZ_CUDA_TRY(cudaEventRecord(t->reps[r]->ev, S(r)));
    }
    RZ_CUDA_TRY(on(0));
    for (int r = 1; r < n; ++r) {
        if (!nr(r)) continue;
        rz_trainer* p = t->reps[r];
        RZ_CUDA_TRY(cudaStreamWaitEvent(st, p->ev, 0));
        const size_t o = b0(r), k = nr(r), fb = sizeof(float);
        RZ_CUDA_TRY(peer(t->hp + o * 128, 0, p->hp, r, k * 128 * fb, st));
        RZ_CUDA_TRY(peer(t->hv + o * 64, 0, p->hv, r, k * 64 * fb, st));
        RZ_CUDA_TRY(peer(t->dl + o * 64, 0, p->dl, r, k * 64 * fb, st));
        RZ_CUDA_TRY(peer(t->h1 + o * V, 0, p->h1, r, k * V * fb, st));
        RZ_CUDA_TRY(peer(t->dh1 + o * V, 0, p->dh1, r, k * V * fb, st));
        RZ_CUDA_TRY(peer(t->dv + o, 0, p->dv, r, k * fb, st));
        RZ_CUDA_TRY(peer(t->lp + o, 0, p->lp, r, k * fb, st));
        RZ_CUDA_TRY(peer(t->lv + o, 0, p->lv, r, k * fb, st));
    }
    const int n_fc = 128 * 64 + 64 + 64 * V + 2 * V + 2;
    head_fc_grad_kernel<<<(n_fc + 255) / 256, 256, 0, st>>>(t->hp, t->hv, t->dl, t->h1, t->dh1, t->dv, t->lp, t->lv, V, batch, t->ho,
                                                            t->grad, t->loss_pv);
    RZ_LAUNCH_CHECK();
    RZ_TRY(bn_backward(dh, ah, hc, 3, 2, bpc, L, dyh, none));
    RZ_TRY(bn_backward(value(dh), value(ah), value(hc), 3, 1, bvc, L + 1, value(dyh), none));
    RZ_TRY(partial_each([&](int, rz_trainer* p, int M, cudaStream_t s) {
        colred_partial_kernel<kHeadConvGrad><<<chunks_of(M), 256, 0, s>>>(at(p, tower), nullptr, p->dyh, F, 3, F, M, nullptr, nullptr, p->part);
    }));
    RZ_TRY(gather_part(3 * (size_t)F));
    colred_finalize_kernel<kHeadConvGrad><<<(F + 255) / 256, 256, 0, st>>>(t->part, chunks, F, Mg, BnRef{t->off_pc, t->off_vc, F}, nullptr,
                                                                           nullptr, nullptr, t->stat, t->grad);
    RZ_LAUNCH_CHECK();
    RZ_TRY(release(-1, 0, 0));
    RZ_TRY(partial_each([&](int, rz_trainer* p, int M, cudaStream_t s) {
        head_conv_dgrad_kernel<<<grid_for((size_t)M * F), 256, 0, s>>>(p->dyh, p->blob, t->off_pc, t->off_vc, F, M, p->g);
    }));

    // tower backward; g holds the gradient of the current block's output
    auto tower_wgrad = [&](int l, Operand in) -> int {
        for (int r = 0; r < n; ++r) {
            if (!nr(r)) continue;
            RZ_CUDA_TRY(on(r));
            rz_trainer* p = t->reps[r];
            RZ_TRY(wgrad(l, r, at(p, in), p->dy, nr(r), b0(r) / per, (nr(r) + per - 1) / per));
        }
        return RZ_OK;
    };
    auto dgrad = [&](int l, Operand add, Operand out) {
        return partial_each([&](int, rz_trainer* p, int M, cudaStream_t s) {
            return launch_conv(p->dy, F, p->wt + (size_t)(l - 1) * 9 * F * F, F, nullptr, at(p, add), at(p, out), M, s);
        });
    };
    for (int i = R - 1; i >= 0; --i) {
        const int l1 = 1 + 2 * i, l2 = l1 + 1;
        RZ_TRY(bn_backward(g, A(l2), Y(l2), F, F, bnref(l2), l2, dy, dz));
        RZ_TRY(tower_wgrad(l2, A(l1)));
        RZ_TRY(dgrad(l2, none, g1));
        RZ_TRY(bn_backward(g1, A(l1), Y(l1), F, F, bnref(l1), l1, dy, none));
        RZ_TRY(tower_wgrad(l1, A(l1 - 1)));
        RZ_TRY(dgrad(l1, dz, g));
    }
    RZ_TRY(bn_backward(g, A(0), Y(0), F, F, bnref(0), 0, dy, none));
    // conv0: a split that straddles the end of shard r takes the first rows of layer 0's dy from replica r + 1 (the x0
    // rows came with the replica's own records)
    Conv0Share c0[64];
    for (int r = 0; r < n; ++r) c0[r] = conv0_share(F, batch, b0(r), nr(r));
    for (int r = 1; r < n; ++r) {
        RZ_CUDA_TRY(on(r));
        const int ov = c0[r - 1].ov;
        if (ov) RZ_CUDA_TRY(peer(t->reps[r - 1]->dy + (size_t)nr(r - 1) * 64 * F, r - 1, t->reps[r]->dy, r, (size_t)ov * 64 * F * sizeof(float),
                                 S(r)));
        RZ_CUDA_TRY(cudaEventRecord(t->reps[r]->ev, S(r)));
    }
    for (int r = 0; r < n; ++r) {
        if (!c0[r].nz) continue;
        RZ_CUDA_TRY(on(r));
        rz_trainer* p = t->reps[r];
        if (c0[r].ov) RZ_CUDA_TRY(cudaStreamWaitEvent(S(r), t->reps[r + 1]->ev, 0));
        RZ_TRY(wgrad(0, r, p->x0 + (size_t)c0[r].row0 * 64 * kCin0, p->dy + (size_t)c0[r].row0 * 64 * F, c0[r].rows, c0[r].z0, c0[r].nz));
    }

    if (n > 1) {  // join the replicas' partials, reduce every layer in split order, hand the gradient out, update the replicas
        for (int r = 1; r < n; ++r) {
            RZ_CUDA_TRY(on(r));
            RZ_CUDA_TRY(cudaEventRecord(t->reps[r]->ev, S(r)));
        }
        RZ_CUDA_TRY(on(0));
        for (int r = 1; r < n; ++r) RZ_CUDA_TRY(cudaStreamWaitEvent(st, t->reps[r]->ev, 0));
        for (int l = 0; l < L; ++l) {
            const int cin = l ? F : kCin0, pl = l ? per : per0;
            wgrad_reduce_kernel<<<grid_for((size_t)9 * cin * F), 256, 0, st>>>(t->wgather + (size_t)l * t->wslot, (batch + pl - 1) / pl, cin,
                                                                               l ? F : 2, F, t->grad + t->conv_off[l]);
        }
        RZ_LAUNCH_CHECK();
        RZ_CUDA_TRY(cudaEventRecord(t->ev, st));
        for (int r = 1; r < n; ++r) {
            rz_trainer* p = t->reps[r];
            RZ_CUDA_TRY(on(r));
            RZ_CUDA_TRY(cudaStreamWaitEvent(p->stream, t->ev, 0));
            RZ_CUDA_TRY(peer(p->grad, r, t->grad, 0, t->n * sizeof(float), p->stream));
            RZ_CUDA_TRY(peer(p->bad, r, t->bad, 0, sizeof(int), p->stream));
            update_kernel<<<kUpdateBlocks, 256, 0, p->stream>>>(p->blob, p->vel, p->grad, p->stat, p->kind, t->n, lr, t->cfg.momentum,
                                                                t->cfg.l2_reg, t->cfg.bn_momentum, p->bad, p->l2_part);
            RZ_LAUNCH_CHECK();
            RZ_CUDA_TRY(cudaEventRecord(p->ev, p->stream));
        }
        RZ_CUDA_TRY(on(0));
        for (int r = 1; r < n; ++r) RZ_CUDA_TRY(cudaStreamWaitEvent(st, t->reps[r]->ev, 0));  // update_kernel rewrites grad
    }
    update_kernel<<<kUpdateBlocks, 256, 0, st>>>(t->blob, t->vel, t->grad, t->stat, t->kind, t->n, lr, t->cfg.momentum, t->cfg.l2_reg,
                                                  t->cfg.bn_momentum, t->bad, t->l2_part);
    loss_kernel<<<1, 32, 0, st>>>(t->l2_part, t->loss_pv, t->cfg.l2_reg, t->bad, loss);
    RZ_LAUNCH_CHECK();
    return RZ_OK;
}

int check_cfg(const rz_net_cfg* net, const rz_train_cfg* cfg) {
    RZ_REQUIRE(net->kernel_size == 3, "trainer: only cnn_filter_size == 3 is supported (got %d)", net->kernel_size);
    RZ_REQUIRE(net->filters >= 16 && net->filters <= 256 && net->filters % 16 == 0,
               "trainer: cnn_filter_num must be a multiple of 16 in [16, 256] (got %d)", net->filters);
    RZ_REQUIRE(net->res_blocks >= 0 && net->res_blocks <= 64 && net->value_fc >= 1 && net->value_fc <= 4096,
               "trainer: unsupported model configuration (res_blocks=%d value_fc=%d)", net->res_blocks, net->value_fc);
    RZ_REQUIRE(cfg->max_batch >= 1 && cfg->max_batch <= 65536, "trainer: max_batch must be in [1, 65536] (got %d)", cfg->max_batch);
    RZ_REQUIRE(isfinite(cfg->momentum) && isfinite(cfg->l2_reg) && isfinite(cfg->bn_momentum), "trainer: non-finite setting");
    return RZ_OK;
}

// A trainer, or one replica of a group: activation and backward buffers for `act` records, the batch-wide buffers (column
// partials, per-record head tensors, staged records) for `full`.  A single trainer has act = full = max_batch and, with
// no replica to exchange with, no staged records, identity index, gradient slots, stream or event.
int trainer_create(const rz_net_cfg* net, const rz_train_cfg* cfg, int device, size_t act, size_t full, bool group, bool primary,
                   rz_trainer** out) {
    RZ_CUDA_TRY(cudaSetDevice(device));
    rz_trainer* t = new (std::nothrow) rz_trainer();
    if (!t) { set_error("out of host memory"); return RZ_ENOMEM; }
    t->net = *net;
    t->cfg = *cfg;
    t->device = device;
    t->act = act;
    const int F = net->filters, R = net->res_blocks, V = net->value_fc;
    t->F = F; t->R = R; t->V = V; t->L = 1 + 2 * R;
    // blob layout of rz_net_load_weights (include/rz_engine.h), with the kind of every entry
    std::vector<uint8_t> kind;
    auto conv_group = [&](size_t kf, int cout) {
        const size_t off = kind.size();
        kind.insert(kind.end(), kf, kKernel);
        kind.insert(kind.end(), (size_t)3 * cout, kTrainable);  // bias, gamma, beta
        kind.insert(kind.end(), (size_t)cout, kMovingMean);
        kind.insert(kind.end(), (size_t)cout, kMovingVar);
        return off;
    };
    t->conv_off.push_back(conv_group((size_t)9 * 2 * F, F));
    for (int l = 1; l < t->L; ++l) t->conv_off.push_back(conv_group((size_t)9 * F * F, F));
    t->off_pc = conv_group((size_t)F * 2, 2);
    t->ho.pfk = kind.size(); kind.insert(kind.end(), 128 * 64, kKernel);
    t->ho.pfb = kind.size(); kind.insert(kind.end(), 64, kTrainable);
    t->off_vc = conv_group((size_t)F, 1);
    t->ho.v1k = kind.size(); kind.insert(kind.end(), (size_t)64 * V, kKernel);
    t->ho.v1b = kind.size(); kind.insert(kind.end(), (size_t)V, kTrainable);
    t->ho.v2k = kind.size(); kind.insert(kind.end(), (size_t)V, kKernel);
    t->ho.v2b = kind.size(); kind.insert(kind.end(), 1, kTrainable);
    t->n = kind.size();

    const size_t B = full, M = 64 * act, MF = M * F, L = t->L;
    const int splits = wgrad_splits(F, F, cfg->max_batch), splits0 = wgrad_splits(kCin0, F, cfg->max_batch);
    t->wslot = std::max((size_t)splits * 9 * F * F, (size_t)splits0 * 9 * kCin0 * F);
    struct { float** p; size_t n; } allocs[] = {
        {&t->blob, t->n}, {&t->vel, t->n}, {&t->grad, t->n}, {&t->stat, t->n}, {&t->x0, M * kCin0}, {&t->w0p, (size_t)9 * kCin0 * F},
        {&t->wt, (size_t)std::max(2 * R, 1) * 9 * F * F}, {&t->y, L * MF}, {&t->a, L * MF}, {&t->g, MF}, {&t->g1, MF}, {&t->dy, MF},
        {&t->dz, MF}, {&t->hc, M * 3}, {&t->ah, M * 3}, {&t->dh, M * 3}, {&t->dyh, M * 3}, {&t->hp, B * 128}, {&t->hv, B * 64},
        {&t->dl, B * 64}, {&t->h1, B * V}, {&t->dh1, B * V}, {&t->dv, B}, {&t->lp, B}, {&t->lv, B}, {&t->stats, (L + 2) * 4 * F},
        {&t->wpart, t->wslot}, {&t->l2_part, kUpdateBlocks}, {&t->loss_pv, 2}};
    cudaError_t e = cudaSuccess;
    for (auto& a : allocs)
        if (e == cudaSuccess) e = cudaMalloc(a.p, a.n * sizeof(float));
    if (group) {
        if (e == cudaSuccess) e = cudaMalloc(&t->sp, B * 128);
        if (e == cudaSuccess) e = cudaMalloc(&t->spol, B * 64 * sizeof(float));
        if (e == cudaSuccess) e = cudaMalloc(&t->sz, B * sizeof(float));
        if (e == cudaSuccess) e = cudaEventCreateWithFlags(&t->ev, cudaEventDisableTiming);
        if (e == cudaSuccess && primary) e = cudaMalloc(&t->wgather, L * t->wslot * sizeof(float));
    }
    if (group && !primary) {
        std::vector<int32_t> iota(act);
        for (size_t i = 0; i < act; ++i) iota[i] = (int32_t)i;
        if (e == cudaSuccess) e = cudaMalloc(&t->iota, act * sizeof(int32_t));
        if (e == cudaSuccess) e = cudaMemcpy(t->iota, iota.data(), act * sizeof(int32_t), cudaMemcpyHostToDevice);
        if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&t->stream, cudaStreamNonBlocking);
    }
    if (e == cudaSuccess) e = cudaMalloc(&t->part, B * 3 * F * sizeof(double));
    if (e == cudaSuccess) e = cudaMalloc(&t->kind, t->n);
    if (e == cudaSuccess) e = cudaMalloc(&t->bad, sizeof(int));
    if (e == cudaSuccess) e = cudaMemcpy(t->kind, kind.data(), t->n, cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = cudaMemset(t->vel, 0, t->n * sizeof(float));
    if (e == cudaSuccess) e = cudaMemset(t->grad, 0, t->n * sizeof(float));
    if (e == cudaSuccess) e = cudaMemset(t->stat, 0, t->n * sizeof(float));
    const size_t fc_smem = head_fc_smem(V);
    if (e == cudaSuccess && fc_smem > 48 * 1024)
        e = cudaFuncSetAttribute(head_fc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)fc_smem);
    if (e != cudaSuccess) {
        set_error("rz_trainer_create: %s", cudaGetErrorString(e));
        cudaGetLastError();
        trainer_free(t);
        delete t;
        return RZ_ENOMEM;
    }
    if (primary) t->reps.push_back(t);
    *out = t;
    return RZ_OK;
}

void trainer_delete(rz_trainer* t) {
    for (size_t r = 1; r < t->reps.size(); ++r) trainer_delete(t->reps[r]);
    cudaSetDevice(t->device);
    trainer_free(t);
    delete t;
}

}  // namespace

extern "C" {

int rz_train_shard_plan_host(int filters, int res_blocks, int batch, int n_devices, int32_t* bounds) {
    RZ_REQUIRE(bounds, "rz_train_shard_plan_host: null pointer");
    RZ_REQUIRE(filters >= 16 && filters <= 256 && filters % 16 == 0 && res_blocks >= 0 && batch >= 1 && n_devices >= 1 && n_devices <= 64,
               "rz_train_shard_plan_host: bad arguments");
    int b[65];
    shard_plan(filters, res_blocks, batch, n_devices, b);
    for (int r = 0; r <= n_devices; ++r) bounds[r] = b[r];
    return RZ_OK;
}

int rz_trainer_create(const rz_net_cfg* net, const rz_train_cfg* cfg, int device, rz_trainer** out) {
    RZ_REQUIRE(net && cfg && out, "rz_trainer_create: null pointer");
    RZ_TRY(check_cfg(net, cfg));
    return trainer_create(net, cfg, device, cfg->max_batch, cfg->max_batch, false, true, out);
}

int rz_trainer_create_group(const rz_net_cfg* net, const rz_train_cfg* cfg, const int* devices, int n_devices, rz_trainer** out) {
    RZ_REQUIRE(net && cfg && devices && out, "rz_trainer_create_group: null pointer");
    RZ_REQUIRE(n_devices >= 1 && n_devices <= 64, "rz_trainer_create_group: n_devices must be in [1, 64] (got %d)", n_devices);
    int count = 0;
    RZ_CUDA_TRY(cudaGetDeviceCount(&count));
    for (int r = 0; r < n_devices; ++r)
        RZ_REQUIRE(devices[r] >= 0 && devices[r] < count, "rz_trainer_create_group: device %d is not one of the %d visible devices",
                   devices[r], count);
    if (n_devices == 1) return rz_trainer_create(net, cfg, devices[0], out);
    RZ_TRY(check_cfg(net, cfg));
    // each replica's largest shard over every batch it can be given, with the records of conv0's straddling split
    std::vector<size_t> act(n_devices, 1);
    int b[65];
    for (int batch = 1; batch <= cfg->max_batch; ++batch) {
        shard_plan(net->filters, net->res_blocks, batch, n_devices, b);
        for (int r = 0; r < n_devices; ++r) {
            const int len = b[r + 1] - b[r], ov = conv0_share(net->filters, batch, b[r], len).ov;
            act[r] = std::max(act[r], (size_t)(len + ov));
        }
    }
    rz_trainer* t = nullptr;
    RZ_TRY(trainer_create(net, cfg, devices[0], act[0], cfg->max_batch, true, true, &t));
    for (int r = 1; r < n_devices; ++r) {
        rz_trainer* p = nullptr;
        const int rc = trainer_create(net, cfg, devices[r], act[r], act[r], true, false, &p);
        if (rc != RZ_OK) {
            trainer_delete(t);
            cudaSetDevice(devices[0]);
            return rc;
        }
        t->reps.push_back(p);
    }
    RZ_CUDA_TRY(cudaSetDevice(devices[0]));
    *out = t;
    return RZ_OK;
}

int rz_trainer_destroy(rz_trainer* t) {
    if (!t) return RZ_OK;
    trainer_delete(t);
    return RZ_OK;
}

int rz_trainer_blob_size(const rz_trainer* t, size_t* n_floats) {
    RZ_REQUIRE(t && n_floats, "rz_trainer_blob_size: null pointer");
    *n_floats = t->n;
    return RZ_OK;
}

int rz_trainer_load_weights(rz_trainer* t, const float* blob_host, size_t n_floats) {
    RZ_REQUIRE(t && blob_host, "rz_trainer_load_weights: null pointer");
    RZ_REQUIRE(n_floats == t->n, "weight blob has %zu floats, this configuration needs %zu", n_floats, t->n);
    for (rz_trainer* p : t->reps) {
        RZ_CUDA_TRY(cudaSetDevice(p->device));
        RZ_CUDA_TRY(cudaMemcpy(p->blob, blob_host, n_floats * sizeof(float), cudaMemcpyHostToDevice));
        RZ_CUDA_TRY(cudaMemset(p->vel, 0, n_floats * sizeof(float)));
    }
    RZ_CUDA_TRY(cudaSetDevice(t->device));
    t->loaded = true;
    return RZ_OK;
}

int rz_trainer_load_weights_dev(rz_trainer* t, const float* blob_dev, size_t n_floats, void* stream) {
    RZ_REQUIRE(t && blob_dev, "rz_trainer_load_weights_dev: null pointer");
    RZ_REQUIRE(n_floats == t->n, "weight blob has %zu floats, this configuration needs %zu", n_floats, t->n);
    RZ_CUDA_TRY(cudaSetDevice(t->device));
    RZ_CUDA_TRY(cudaMemcpyAsync(t->blob, blob_dev, n_floats * sizeof(float), cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
    RZ_CUDA_TRY(cudaMemsetAsync(t->vel, 0, n_floats * sizeof(float), (cudaStream_t)stream));
    for (size_t r = 1; r < t->reps.size(); ++r) {  // the replicas copy the primary, in the caller's stream order
        rz_trainer* p = t->reps[r];
        RZ_CUDA_TRY(cudaMemcpyPeerAsync(p->blob, p->device, t->blob, t->device, n_floats * sizeof(float), (cudaStream_t)stream));
        RZ_CUDA_TRY(cudaMemcpyPeerAsync(p->vel, p->device, t->vel, t->device, n_floats * sizeof(float), (cudaStream_t)stream));
    }
    t->loaded = true;
    return RZ_OK;
}

int rz_trainer_weights_dev(rz_trainer* t, float* blob_dev, size_t n_floats, void* stream) {
    RZ_REQUIRE(t && blob_dev, "rz_trainer_weights_dev: null pointer");
    RZ_REQUIRE(n_floats == t->n, "weight blob has %zu floats, this configuration needs %zu", n_floats, t->n);
    if (!t->loaded) { set_error("rz_trainer: weights not loaded"); return RZ_ESTATE; }
    RZ_CUDA_TRY(cudaSetDevice(t->device));
    RZ_CUDA_TRY(cudaMemcpyAsync(blob_dev, t->blob, n_floats * sizeof(float), cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
    return RZ_OK;
}

int rz_trainer_step_dev(rz_trainer* t, const uint8_t* planes, const float* policy, const float* z, size_t n_records,
                        const int32_t* index, size_t batch, float lr, float* loss_dev, void* stream) {
    RZ_REQUIRE(t && planes && policy && z && index && loss_dev, "rz_trainer_step_dev: null pointer");
    RZ_REQUIRE(batch >= 1 && batch <= (size_t)t->cfg.max_batch, "batch %zu outside [1, max_batch = %d]", batch, t->cfg.max_batch);
    RZ_REQUIRE(n_records >= 1, "rz_trainer_step_dev: empty dataset");
    RZ_REQUIRE(isfinite(lr), "rz_trainer_step_dev: non-finite learning rate");
    if (!t->loaded) { set_error("rz_trainer: weights not loaded"); return RZ_ESTATE; }
    RZ_CUDA_TRY(cudaSetDevice(t->device));
    const int rc = step(t, planes, policy, z, index, n_records, (int)batch, lr, loss_dev, (cudaStream_t)stream);
    cudaSetDevice(t->device);
    return rc;
}

int rz_trainer_replica_state_dev(rz_trainer* t, int r, float* blob_dev, float* vel_dev, size_t n_floats, void* stream) {
    RZ_REQUIRE(t && blob_dev && vel_dev, "rz_trainer_replica_state_dev: null pointer");
    RZ_REQUIRE(n_floats == t->n, "weight blob has %zu floats, this configuration needs %zu", n_floats, t->n);
    const int n = (int)t->reps.size();
    RZ_REQUIRE(r >= 0 && r < n, "rz_trainer_replica_state_dev: replica %d outside [0, %d)", r, n);
    const rz_trainer* p = t->reps[r];
    RZ_CUDA_TRY(cudaSetDevice(t->device));
    RZ_CUDA_TRY(cudaMemcpyPeerAsync(blob_dev, t->device, p->blob, p->device, n_floats * sizeof(float), (cudaStream_t)stream));
    RZ_CUDA_TRY(cudaMemcpyPeerAsync(vel_dev, t->device, p->vel, p->device, n_floats * sizeof(float), (cudaStream_t)stream));
    return RZ_OK;
}

int rz_trainer_last_grad_dev(rz_trainer* t, float* grad_dev, size_t n_floats, void* stream) {
    RZ_REQUIRE(t && grad_dev, "rz_trainer_last_grad_dev: null pointer");
    RZ_REQUIRE(n_floats == t->n, "gradient has %zu floats, this configuration needs %zu", n_floats, t->n);
    RZ_CUDA_TRY(cudaSetDevice(t->device));
    mask_grad_kernel<<<grid_for(t->n), 256, 0, (cudaStream_t)stream>>>(t->grad, t->kind, t->n, grad_dev);
    RZ_LAUNCH_CHECK();
    return RZ_OK;
}

int rz_trainer_debug_conv_dev(rz_trainer* t, int op, const float* in, const float* kernel, const float* bias, const float* add,
                              size_t batch, float* out, void* stream) {
    RZ_REQUIRE(t && in && out, "rz_trainer_debug_conv_dev: null pointer");
    RZ_REQUIRE(batch >= 1 && batch <= (size_t)t->cfg.max_batch, "batch %zu outside [1, max_batch = %d]", batch, t->cfg.max_batch);
    const int F = t->F, M = (int)batch * 64;
    const cudaStream_t st = (cudaStream_t)stream;
    RZ_CUDA_TRY(cudaSetDevice(t->device));
    switch (op) {
        case RZ_TRAIN_CONV0_FWD:
            RZ_REQUIRE(kernel, "rz_trainer_debug_conv_dev: null kernel");
            pack_w0_kernel<<<(9 * kCin0 * F + 255) / 256, 256, 0, st>>>(kernel, F, t->w0p);
            RZ_LAUNCH_CHECK();
            return launch_conv(in, kCin0, t->w0p, F, bias, add, out, M, st);
        case RZ_TRAIN_CONV_FWD:
            RZ_REQUIRE(kernel, "rz_trainer_debug_conv_dev: null kernel");
            return launch_conv(in, F, kernel, F, bias, add, out, M, st);
        case RZ_TRAIN_CONV_DGRAD:
            RZ_REQUIRE(kernel, "rz_trainer_debug_conv_dev: null kernel");
            pack_wt_kernel<<<grid_for((size_t)9 * F * F), 256, 0, st>>>(kernel, F, t->wt);
            RZ_LAUNCH_CHECK();
            return launch_conv(in, F, t->wt, F, bias, add, out, M, st);
        case RZ_TRAIN_CONV_WGRAD:
        case RZ_TRAIN_CONV0_WGRAD: {
            RZ_REQUIRE(add && !kernel && !bias, "rz_trainer_debug_conv_dev: the weight gradient takes dy in `add`, no kernel or bias");
            const bool c0 = op == RZ_TRAIN_CONV0_WGRAD;  // all of the layer's splits at this batch, reduced at once as in the step
            const int cin = c0 ? kCin0 : F, per = wgrad_per(cin, F, (int)batch);
            return launch_wgrad(in, cin, c0 ? 2 : F, add, F, (int)batch, ((int)batch + per - 1) / per, per, t->wpart, out, st);
        }
        default:
            set_error("rz_trainer_debug_conv_dev: unknown op %d", op);
            return RZ_EINVAL;
    }
}

int rz_trainer_debug_keep_backward(rz_trainer* t, int on) {
    RZ_REQUIRE(t, "rz_trainer_debug_keep_backward: null pointer");
    if (t->reps.size() > 1) { set_error("rz_trainer_debug_keep_backward: not available on a data-parallel group"); return RZ_ESTATE; }
    RZ_CUDA_TRY(cudaSetDevice(t->device));
    t->taps_valid = false;
    if (!on) {
        RZ_CUDA_TRY(cudaFree(t->taps));
        t->taps = nullptr;
        return RZ_OK;
    }
    if (t->taps) return RZ_OK;
    const size_t n = (size_t)t->L * 3 * 64 * t->act * t->F;
    if (cudaMalloc(&t->taps, n * sizeof(float)) != cudaSuccess) {
        cudaGetLastError();
        t->taps = nullptr;
        set_error("rz_trainer_debug_keep_backward: cannot allocate %zu floats", n);
        return RZ_ENOMEM;
    }
    RZ_CUDA_TRY(cudaMemset(t->taps, 0, n * sizeof(float)));
    return RZ_OK;
}

int rz_trainer_debug_tensor_dev(rz_trainer* t, int which, int layer, float* out, size_t n_floats, void* stream) {
    RZ_REQUIRE(t && out, "rz_trainer_debug_tensor_dev: null pointer");
    if (t->reps.size() > 1) { set_error("rz_trainer_debug_tensor_dev: not available on a data-parallel group"); return RZ_ESTATE; }
    if (!t->last_batch) { set_error("rz_trainer_debug_tensor_dev: no step has run"); return RZ_ESTATE; }
    const size_t B = t->last_batch, M = 64 * B, F = t->F, V = t->V, stride = 64 * t->act * F;
    const bool tower = which == RZ_TRAIN_T_Y || which == RZ_TRAIN_T_A || which >= RZ_TRAIN_T_G;
    const int layers = tower ? t->L : which == RZ_TRAIN_T_STATS ? t->L + 2 : 1;
    RZ_REQUIRE(which >= 0 && which <= RZ_TRAIN_T_DZ, "rz_trainer_debug_tensor_dev: unknown tensor %d", which);
    RZ_REQUIRE(layer >= 0 && layer < layers, "rz_trainer_debug_tensor_dev: layer %d outside [0, %d) for tensor %d", layer, layers, which);
    RZ_REQUIRE(which != RZ_TRAIN_T_DZ || (layer >= 2 && layer % 2 == 0), "rz_trainer_debug_tensor_dev: layer %d keeps no dz", layer);
    if (which >= RZ_TRAIN_T_G && !t->taps_valid) {
        set_error("rz_trainer_debug_tensor_dev: the last step ran without rz_trainer_debug_keep_backward");
        return RZ_ESTATE;
    }
    const float* src = nullptr;
    size_t count = 0;
    switch (which) {
        case RZ_TRAIN_T_X0: src = t->x0; count = M * kCin0; break;
        case RZ_TRAIN_T_Y: src = t->y + layer * stride; count = M * F; break;
        case RZ_TRAIN_T_A: src = t->a + layer * stride; count = M * F; break;
        case RZ_TRAIN_T_STATS: src = t->stats + (size_t)layer * 4 * F; count = 4 * F; break;
        case RZ_TRAIN_T_STAT: src = t->stat; count = t->n; break;
        case RZ_TRAIN_T_HC: src = t->hc; count = M * 3; break;
        case RZ_TRAIN_T_AH: src = t->ah; count = M * 3; break;
        case RZ_TRAIN_T_DH: src = t->dh; count = M * 3; break;
        case RZ_TRAIN_T_DYH: src = t->dyh; count = M * 3; break;
        case RZ_TRAIN_T_HP: src = t->hp; count = B * 128; break;
        case RZ_TRAIN_T_HV: src = t->hv; count = B * 64; break;
        case RZ_TRAIN_T_DL: src = t->dl; count = B * 64; break;
        case RZ_TRAIN_T_H1: src = t->h1; count = B * V; break;
        case RZ_TRAIN_T_DH1: src = t->dh1; count = B * V; break;
        case RZ_TRAIN_T_DV: src = t->dv; count = B; break;
        case RZ_TRAIN_T_LP: src = t->lp; count = B; break;
        case RZ_TRAIN_T_LV: src = t->lv; count = B; break;
        case RZ_TRAIN_T_LOSS_PV: src = t->loss_pv; count = 2; break;
        default: src = t->taps + ((size_t)layer * 3 + (which - RZ_TRAIN_T_G)) * stride; count = M * F; break;  // G, DY, DZ
    }
    RZ_REQUIRE(n_floats == count, "rz_trainer_debug_tensor_dev: tensor %d has %zu floats, got %zu", which, count, n_floats);
    RZ_CUDA_TRY(cudaSetDevice(t->device));
    RZ_CUDA_TRY(cudaMemcpyAsync(out, src, count * sizeof(float), cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
    return RZ_OK;
}

}  // extern "C"
