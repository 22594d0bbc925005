// rz_ingest_json.cu -- trainer-side ingest of play_*.json text on the device: what the reference trainer does with
// json.load (lib/data_helper.py:28-30) and OptimizeWorker.convert_to_training_data (worker/optimize.py:215-231), for
// files written by the reference's own self-play or by this engine without the play_*.rzrows twin.
//
// Two passes over the text, which is already in device memory:
//   index  json_depth_kernel     per 4 KB tile: the bracket-depth change, and any '"' (the format has no strings)
//          (CUB exclusive scan of the tile depths)
//          json_starts_kernel    per byte the depth before it; a '[' entered from depth 1 opens a record.  Counted per
//                                tile, scanned, one host read of the record count, then the same kernel writes the starts
//   parse  json_parse_kernel     one warp per record: 32 bytes per step, items found with a ballot, each number parsed
//                                by the lane its first byte falls on (rz_json_parse.cuh), stores as in ingest_kernel
// Every byte of the text is checked: the head before the first record ("["), each record against the fixed 139-item
// skeleton, the gap after it ("," or, after the last, "]"), with whitespace anywhere.  The reported error is the
// smallest offset any check finds, the same one the host twin reports.
//
// Numbers: Clinger's fast path and Eisel-Lemire on the device.  What they leave open (more than 19 significant digits,
// subnormal / zero / infinite results, products too close to a halfway point) flags the record; the host then copies
// that record's text back, converts it with the exact strtod of the C library and patches the record's policy and z.
#include <errno.h>
#include <locale.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <string>
#include <vector>
#include <cub/cub.cuh>
#include "rz_common.cuh"
#include "rz_json_parse.cuh"

namespace rz {
using json::u64;
using json::kNoError;

constexpr int kTileBytes = 4096;
constexpr int kScanThreads = 256;  // 16 bytes per thread
constexpr int kParseThreads = 256;
constexpr int kParseWarps = kParseThreads / 32;

__device__ const u64 d_pow10[RZ_POW10_MAX_E - RZ_POW10_MIN_E + 1][2] = RZ_POW10_TABLE_INIT;
static const u64 h_pow10[RZ_POW10_MAX_E - RZ_POW10_MIN_E + 1][2] = RZ_POW10_TABLE_INIT;

struct JsonFallback { u64 record, begin, end; };  // a record whose numbers need the exact conversion

__device__ __forceinline__ void load16(const unsigned char* text, u64 off, u64 n, bool aligned, unsigned char b[16]) {
    if (aligned && off + 16 <= n) {
        const uint4 v = __ldg(reinterpret_cast<const uint4*>(text + off));
        memcpy(b, &v, 16);
    } else {
#pragma unroll
        for (int i = 0; i < 16; ++i) b[i] = off + i < n ? text[off + i] : (unsigned char)' ';
    }
}

__device__ __forceinline__ void error_at(unsigned long long* err, u64 off) { atomicMin(err, (unsigned long long)off); }

__global__ void __launch_bounds__(kScanThreads) json_depth_kernel(const unsigned char* __restrict__ text, u64 n, bool aligned,
                                                                  int* __restrict__ tile_delta, unsigned long long* err) {
    typedef cub::BlockReduce<int, kScanThreads> Reduce;
    __shared__ typename Reduce::TempStorage tmp;
    const u64 off = (u64)blockIdx.x * kTileBytes + threadIdx.x * 16;
    unsigned char b[16];
    load16(text, off, n, aligned, b);
    int d = 0;
#pragma unroll
    for (int i = 0; i < 16; ++i) {
        d += (b[i] == '[') - (b[i] == ']');
        if (b[i] == '"') error_at(err, off + i);
    }
    d = Reduce(tmp).Sum(d);
    if (threadIdx.x == 0) tile_delta[blockIdx.x] = d;
}

// WRITE = false: tile_records[t] = number of records starting in tile t.  WRITE = true: starts[tile_first[t] + k] = the
// byte offset of the tile's k-th record.
template <bool WRITE>
__global__ void __launch_bounds__(kScanThreads) json_starts_kernel(const unsigned char* __restrict__ text, u64 n, bool aligned,
                                                                   const int* __restrict__ tile_depth, u64* __restrict__ tile_records,
                                                                   u64* __restrict__ starts) {
    typedef cub::BlockScan<int, kScanThreads> Scan;
    __shared__ typename Scan::TempStorage tmp;
    const u64 off = (u64)blockIdx.x * kTileBytes + threadIdx.x * 16;
    unsigned char b[16];
    load16(text, off, n, aligned, b);
    int d = 0;
#pragma unroll
    for (int i = 0; i < 16; ++i) d += (b[i] == '[') - (b[i] == ']');
    Scan(tmp).ExclusiveSum(d, d);
    d += tile_depth[blockIdx.x];
    const int d0 = d;
    int cnt = 0;
#pragma unroll
    for (int i = 0; i < 16; ++i) {
        cnt += b[i] == '[' && d == 1;
        d += (b[i] == '[') - (b[i] == ']');
    }
    __syncthreads();
    int first, total;
    Scan(tmp).ExclusiveSum(cnt, first, total);
    if (!WRITE) {
        if (threadIdx.x == 0) tile_records[blockIdx.x] = (u64)total;
        return;
    }
    if (!cnt) return;
    u64 k = tile_records[blockIdx.x] + (u64)first;
    d = d0;
#pragma unroll
    for (int i = 0; i < 16; ++i) {
        if (b[i] == '[' && d == 1) starts[k++] = off + i;
        d += (b[i] == '[') - (b[i] == ']');
    }
}

__device__ __forceinline__ u64 warp_min(u64 v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const u64 w = __shfl_xor_sync(0xffffffffu, v, o);
        v = w < v ? w : v;
    }
    return v;
}

// The non-whitespace bytes of text[from, to) must be exactly `pattern`; returns the first offending offset, `to` when
// the pattern is not complete, or kNoError.
__device__ u64 warp_match(const unsigned char* text, u64 from, u64 to, const char* pattern, int plen) {
    const int lane = threadIdx.x & 31;
    int ord = 0;
    for (u64 pos = from; pos < to; pos += 32) {
        const u64 p = pos + lane;
        const unsigned char c = p < to ? text[p] : ' ';
        const bool item = json::byte_class(c) != json::C_WS;
        const unsigned m = __ballot_sync(0xffffffffu, item);
        const int my = ord + __popc(m & ((1u << lane) - 1));
        const u64 e = warp_min(item && (my >= plen || c != (unsigned char)pattern[my]) ? p : kNoError);
        if (e != kNoError) return e;
        ord += __popc(m);
    }
    return ord < plen ? to : kNoError;
}

__device__ __forceinline__ uint32_t bits4_to_bytes_j(uint32_t b) { return (b * 0x00204081u) & 0x01010101u; }

__global__ void __launch_bounds__(kParseThreads, 4) json_parse_kernel(const unsigned char* __restrict__ text, u64 n,
                                                                   const u64* __restrict__ starts, u64 n_rec,
                                                                   uint8_t* __restrict__ planes, float* __restrict__ policy,
                                                                   float* __restrict__ z, unsigned long long* err,
                                                                   JsonFallback* fallback, unsigned long long* n_fallback) {
    __shared__ __align__(16) float pol_s[kParseWarps][64];
    __shared__ u64 brd_s[kParseWarps][2];
    __shared__ float z_s[kParseWarps];
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const unsigned lt = (1u << lane) - 1;
    if (n_rec == 0) {  // the whole text must be an empty array
        if (blockIdx.x == 0 && w == 0) {
            const u64 e = warp_match(text, 0, n, "[]", 2);
            if (lane == 0 && e != kNoError) error_at(err, e);
        }
        return;
    }
    const u64 n_warps = (u64)gridDim.x * kParseWarps;
    for (u64 r = (u64)blockIdx.x * kParseWarps + w; r < n_rec; r += n_warps) {
        const u64 s = starts[r];
        u64 e = kNoError, rec_end = 0, pos = s;
        int ord = 0;
        bool exact_needed = false;
        for (;;) {
            const u64 p = pos + lane;
            const bool in = p < n;
            const unsigned char c = in ? text[p] : ' ';
            unsigned char prev = __shfl_up_sync(0xffffffffu, c, 1);
            if (lane == 0) prev = text[pos - 1];  // pos >= s >= 1: a record is always inside the top-level '['
            const int cls = json::byte_class(c);
            const bool item = cls != json::C_WS && !(cls == json::C_NUM && json::byte_class(prev) == json::C_NUM);
            const unsigned m = __ballot_sync(0xffffffffu, item);
            const int my = ord + __popc(m & lt);
            u64 le = kNoError;
            bool exact = false;
            if (item && my < json::kItems) {  // items past the record's closing bracket belong to the gap after it
                const char k = json::item_kind(my);
                if (k != 'N') {
                    if (c != (unsigned char)k) le = p;
                } else if (cls != json::C_NUM) {
                    le = p;
                } else {
                    const u64 b = json::token_end(text, p, n);
                    if (my == json::kOwnItem || my == json::kEnemyItem) {
                        u64 v;
                        if (json::parse_u64(text, p, b, &v)) brd_s[w][my == json::kEnemyItem] = v;
                        else le = p;
                    } else {
                        double v = 0;
                        const int st = json::parse_number(text, p, b, d_pow10, &v);
                        if (st == json::NUM_BAD) le = p;
                        exact = st == json::NUM_EXACT_NEEDED;
                        const float f = json::to_float32(v);
                        if (my == json::kZItem) z_s[w] = f;
                        else pol_s[w][(my - json::kFirstPolicyItem) >> 1] = f;
                    }
                }
            }
            exact_needed |= __any_sync(0xffffffffu, exact);
            const unsigned closing = __ballot_sync(0xffffffffu, item && my == json::kItems - 1);
            ord += __popc(m);
            e = warp_min(le);
            if (e != kNoError) break;
            if (closing) { rec_end = pos + __ffs(closing); break; }
            if (pos + 32 >= n) { e = n; break; }  // the text ends inside the record
            pos += 32;
        }
        if (e == kNoError) e = warp_match(text, rec_end, r + 1 < n_rec ? starts[r + 1] : n, r + 1 < n_rec ? "," : "]", 1);
        if (r == 0) {
            const u64 h = warp_match(text, 0, s, "[", 1);
            e = h < e ? h : e;
        }
        __syncwarp();
        if (e != kNoError) {
            if (lane == 0) error_at(err, e);
            continue;
        }
        if (lane < 8) {  // planes: 2 x 64 squares, 16 squares per lane (bit_to_array, lib/bitboard.py:136-138)
            const uint32_t bits = (uint32_t)(brd_s[w][lane >> 2] >> (16 * (lane & 3))) & 0xFFFFu;
            const uint4 v = make_uint4(bits4_to_bytes_j(bits & 15u), bits4_to_bytes_j((bits >> 4) & 15u),
                                       bits4_to_bytes_j((bits >> 8) & 15u), bits4_to_bytes_j(bits >> 12));
            __stcs(reinterpret_cast<uint4*>(planes + r * 128) + lane, v);
        } else if (lane < 24) {
            const int q = lane - 8;
            __stcs(reinterpret_cast<float4*>(policy + r * 64) + q, *reinterpret_cast<const float4*>(&pol_s[w][4 * q]));
        } else if (lane == 24) {
            __stcs(z + r, z_s[w]);
        } else if (lane == 25 && exact_needed) {
            const unsigned long long i = atomicAdd(n_fallback, 1ull);
            fallback[i] = JsonFallback{r, s, rec_end};
        }
        __syncwarp();
    }
}

// one fallback record's exact policy and z, from the host
__global__ void json_patch_kernel(const u64* __restrict__ records, const float* __restrict__ values, u64 n, float* __restrict__ policy,
                                  float* __restrict__ z) {
    for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < n * 65; i += (u64)gridDim.x * blockDim.x) {
        const u64 k = i / 65, j = i % 65, r = records[k];
        if (j < 64) policy[r * 64 + j] = values[i];
        else z[r] = values[i];
    }
}

// ---- host side: the twin of the kernels above, and the exact conversion -----------------------------------------
static double exact_decimal(const unsigned char* s, u64 a, u64 b) {
    static locale_t c_locale = newlocale(LC_ALL_MASK, "C", (locale_t)0);
    const std::string tok((const char*)s + a, (size_t)(b - a));
    return strtod_l(tok.c_str(), nullptr, c_locale);  // correctly rounded; overflow gives inf, underflow 0 or a subnormal
}

static u64 host_match(const unsigned char* text, u64 from, u64 to, const char* pattern, int plen) {
    int ord = 0;
    for (u64 p = from; p < to; ++p) {
        if (json::byte_class(text[p]) == json::C_WS) continue;
        if (ord >= plen || text[p] != (unsigned char)pattern[ord]) return p;
        ++ord;
    }
    return ord < plen ? to : kNoError;
}

// The record starting at s: returns kNoError and fills the outputs (exact conversion included), else the first
// offending offset.  *end = the byte after its closing bracket.
static u64 host_record(const unsigned char* text, u64 s, u64 n, uint8_t* planes, float* policy, float* z, u64* end) {
    int ord = 0;
    u64 brd[2] = {0, 0};
    for (u64 p = s; p < n; ++p) {
        const int cls = json::byte_class(text[p]);
        if (cls == json::C_WS || (cls == json::C_NUM && json::byte_class(text[p - 1]) == json::C_NUM)) continue;
        const char k = json::item_kind(ord);
        if (k != 'N') {
            if (text[p] != (unsigned char)k) return p;
        } else if (cls != json::C_NUM) {
            return p;
        } else {
            const u64 b = json::token_end(text, p, n);
            if (ord == json::kOwnItem || ord == json::kEnemyItem) {
                if (!json::parse_u64(text, p, b, &brd[ord == json::kEnemyItem])) return p;
            } else {
                double v = 0;
                const int st = json::parse_number(text, p, b, h_pow10, &v);
                if (st == json::NUM_BAD) return p;
                if (st == json::NUM_EXACT_NEEDED) v = exact_decimal(text, p, b);
                const float f = json::to_float32(v);
                if (ord == json::kZItem) *z = f;
                else policy[(ord - json::kFirstPolicyItem) >> 1] = f;
            }
        }
        if (++ord == json::kItems) {
            *end = p + 1;
            for (int i = 0; i < 128; ++i) planes[i] = (uint8_t)((brd[i >> 6] >> (i & 63)) & 1);
            return kNoError;
        }
    }
    return n;
}

static void host_index(const unsigned char* text, u64 n, std::vector<u64>& starts, u64* err) {
    long long d = 0;
    for (u64 p = 0; p < n; ++p) {
        const unsigned char c = text[p];
        if (c == '"' && p < *err) *err = p;
        if (c == '[' && d == 1) starts.push_back(p);
        d += (c == '[') - (c == ']');
    }
}

static int report(u64 err, size_t* error_offset, const char* who) {
    if (error_offset) *error_offset = err == kNoError ? (size_t)-1 : (size_t)err;
    if (err == kNoError) return RZ_OK;
    set_error("%s: malformed play JSON at byte %llu", who, (unsigned long long)err);
    return RZ_EINVAL;
}

static unsigned parse_blocks(u64 n_rec) {
    u64 blocks = (n_rec + kParseWarps - 1) / kParseWarps;
    const u64 cap = (u64)num_sms() * 16;
    if (blocks > cap) blocks = cap;
    return (unsigned)(blocks ? blocks : 1);
}

}  // namespace rz

using namespace rz;

extern "C" {

int rz_ingest_json_host(const char* text, size_t n_bytes, size_t capacity, uint8_t* planes, float* policy, float* z,
                        size_t* n_records, size_t* error_offset) {
    RZ_REQUIRE(n_records && (n_bytes == 0 || text), "rz_ingest_json_host: null pointer");
    if (error_offset) *error_offset = (size_t)-1;
    const unsigned char* t = (const unsigned char*)text;
    std::vector<u64> starts;
    u64 err = kNoError;
    host_index(t, n_bytes, starts, &err);
    const u64 nr = starts.size();
    *n_records = (size_t)nr;
    if (nr > capacity) {
        set_error("rz_ingest_json_host: %llu records, capacity %zu", (unsigned long long)nr, capacity);
        return RZ_ECAPACITY;
    }
    RZ_REQUIRE(nr == 0 || (planes && policy && z), "rz_ingest_json_host: null pointer");
    if (nr == 0) {
        const u64 e = host_match(t, 0, n_bytes, "[]", 2);
        return report(e < err ? e : err, error_offset, "rz_ingest_json_host");
    }
    const u64 h = host_match(t, 0, starts[0], "[", 1);
    err = h < err ? h : err;
    for (u64 r = 0; r < nr; ++r) {
        u64 end = 0;
        u64 e = host_record(t, starts[r], n_bytes, planes + r * 128, policy + r * 64, z + r, &end);
        if (e == kNoError) e = host_match(t, end, r + 1 < nr ? starts[r + 1] : n_bytes, r + 1 < nr ? "," : "]", 1);
        err = e < err ? e : err;
    }
    return report(err, error_offset, "rz_ingest_json_host");
}

int rz_ingest_json_dev(const char* text, size_t n_bytes, size_t capacity, uint8_t* planes, float* policy, float* z,
                       size_t* n_records, size_t* error_offset, void* stream) {
    RZ_REQUIRE(n_records && (n_bytes == 0 || text), "rz_ingest_json_dev: null pointer");
    if (error_offset) *error_offset = (size_t)-1;
    cudaStream_t st = (cudaStream_t)stream;
    const unsigned char* t = (const unsigned char*)text;
    const bool aligned = ((uintptr_t)text & 15) == 0;
    const u64 n = n_bytes, tiles = (n + kTileBytes - 1) / kTileBytes;
    // scratch: err, n_fallback | tile depth (tiles) | tile records (tiles + 1) | CUB temp
    size_t cub_a = 0, cub_b = 0;
    RZ_CUDA_TRY(cub::DeviceScan::ExclusiveSum(nullptr, cub_a, (int*)nullptr, (int*)nullptr, (int)(tiles + 1), st));
    RZ_CUDA_TRY(cub::DeviceScan::ExclusiveSum(nullptr, cub_b, (u64*)nullptr, (u64*)nullptr, (int)(tiles + 1), st));
    const size_t o_depth = 256, o_rec = o_depth + ((tiles + 1) * sizeof(int) + 255) / 256 * 256,
                 o_cub = o_rec + ((tiles + 1) * sizeof(u64) + 255) / 256 * 256, total = o_cub + (cub_a > cub_b ? cub_a : cub_b);
    char* scratch = nullptr;
    RZ_CUDA_TRY(cudaMallocAsync((void**)&scratch, total, st));
    unsigned long long* d_err = (unsigned long long*)scratch;
    unsigned long long* d_nfb = d_err + 1;
    int* depth = (int*)(scratch + o_depth);
    u64* recs = (u64*)(scratch + o_rec);
    void* cub_tmp = scratch + o_cub;
    u64* starts = nullptr;
    JsonFallback* fb = nullptr;
    int rc = RZ_OK;
    u64 nr = 0, herr = kNoError, nfb = 0;
    cudaError_t ce = cudaMemsetAsync(d_err, 0xFF, 8, st);
    if (ce == cudaSuccess) ce = cudaMemsetAsync(d_nfb, 0, 8, st);
    if (ce == cudaSuccess) ce = cudaMemsetAsync(depth, 0, (tiles + 1) * sizeof(int), st);
    if (ce == cudaSuccess) ce = cudaMemsetAsync(recs, 0, (tiles + 1) * sizeof(u64), st);
    if (ce == cudaSuccess && tiles) {
        json_depth_kernel<<<(unsigned)tiles, kScanThreads, 0, st>>>(t, n, aligned, depth, d_err);
        size_t sz = cub_a;
        ce = cudaGetLastError();
        if (ce == cudaSuccess) ce = cub::DeviceScan::ExclusiveSum(cub_tmp, sz, depth, depth, (int)(tiles + 1), st);
        if (ce == cudaSuccess) json_starts_kernel<false><<<(unsigned)tiles, kScanThreads, 0, st>>>(t, n, aligned, depth, recs, nullptr);
        if (ce == cudaSuccess) ce = cudaGetLastError();
        sz = cub_b;
        if (ce == cudaSuccess) ce = cub::DeviceScan::ExclusiveSum(cub_tmp, sz, recs, recs, (int)(tiles + 1), st);
    }
    if (ce == cudaSuccess) ce = cudaMemcpyAsync(&nr, recs + tiles, sizeof(u64), cudaMemcpyDeviceToHost, st);
    if (ce == cudaSuccess) ce = cudaStreamSynchronize(st);  // the one host read that sizes the outputs
    if (ce == cudaSuccess) {
        *n_records = (size_t)nr;
        if (nr > capacity) {
            set_error("rz_ingest_json_dev: %llu records, capacity %zu", (unsigned long long)nr, capacity);
            rc = RZ_ECAPACITY;
        } else if (nr && !(planes && policy && z)) {
            set_error("rz_ingest_json_dev: null pointer");
            rc = RZ_EINVAL;
        }
    }
    if (ce == cudaSuccess && rc == RZ_OK && nr) {
        ce = cudaMallocAsync((void**)&starts, nr * (sizeof(u64) + sizeof(JsonFallback)), st);
        fb = (JsonFallback*)(starts + nr);
        if (ce == cudaSuccess) json_starts_kernel<true><<<(unsigned)tiles, kScanThreads, 0, st>>>(t, n, aligned, depth, recs, starts);
        if (ce == cudaSuccess) ce = cudaGetLastError();
    }
    if (ce == cudaSuccess && rc == RZ_OK) {
        json_parse_kernel<<<parse_blocks(nr), kParseThreads, 0, st>>>(t, n, starts, nr, planes, policy, z, d_err, fb, d_nfb);
        ce = cudaGetLastError();
        if (ce == cudaSuccess) ce = cudaMemcpyAsync(&herr, d_err, 8, cudaMemcpyDeviceToHost, st);
        if (ce == cudaSuccess) ce = cudaMemcpyAsync(&nfb, d_nfb, 8, cudaMemcpyDeviceToHost, st);
        if (ce == cudaSuccess) ce = cudaStreamSynchronize(st);
    }
    if (ce == cudaSuccess && rc == RZ_OK && herr == kNoError && nfb) {
        // the records the fast paths could not round: their text back to the host, the exact conversion, a patch
        std::vector<JsonFallback> list(nfb);
        ce = cudaMemcpyAsync(list.data(), fb, nfb * sizeof(JsonFallback), cudaMemcpyDeviceToHost, st);
        if (ce == cudaSuccess) ce = cudaStreamSynchronize(st);
        std::vector<std::vector<unsigned char>> texts(nfb);
        for (u64 i = 0; ce == cudaSuccess && i < nfb; ++i) {
            texts[i].resize(list[i].end - list[i].begin);
            ce = cudaMemcpyAsync(texts[i].data(), t + list[i].begin, texts[i].size(), cudaMemcpyDeviceToHost, st);
        }
        if (ce == cudaSuccess) ce = cudaStreamSynchronize(st);
        std::vector<u64> idx(nfb);
        std::vector<float> vals(nfb * 65);
        for (u64 i = 0; ce == cudaSuccess && i < nfb; ++i) {
            uint8_t pl[128];
            u64 end = 0;
            const unsigned char* base = texts[i].data() - list[i].begin;  // indexes as in the whole text
            if (host_record(base, list[i].begin, list[i].end, pl, &vals[i * 65], &vals[i * 65 + 64], &end) != kNoError) {
                set_error("rz_ingest_json_dev: record %llu does not parse on the host", (unsigned long long)list[i].record);
                rc = RZ_ECUDA;
                break;
            }
            idx[i] = list[i].record;
        }
        char* patch = nullptr;
        if (ce == cudaSuccess && rc == RZ_OK) ce = cudaMallocAsync((void**)&patch, nfb * (sizeof(u64) + 65 * sizeof(float)), st);
        if (ce == cudaSuccess && rc == RZ_OK) {
            float* pv = (float*)(patch + nfb * sizeof(u64));
            ce = cudaMemcpyAsync(patch, idx.data(), nfb * sizeof(u64), cudaMemcpyHostToDevice, st);
            if (ce == cudaSuccess) ce = cudaMemcpyAsync(pv, vals.data(), nfb * 65 * sizeof(float), cudaMemcpyHostToDevice, st);
            if (ce == cudaSuccess) {
                json_patch_kernel<<<(unsigned)((nfb * 65 + 255) / 256 < 1024 ? (nfb * 65 + 255) / 256 : 1024), 256, 0, st>>>(
                    (const u64*)patch, pv, nfb, policy, z);
                ce = cudaGetLastError();
            }
            if (ce == cudaSuccess) ce = cudaStreamSynchronize(st);  // the host vectors are the copies' sources
            cudaFreeAsync(patch, st);
        }
    }
    if (starts) cudaFreeAsync(starts, st);
    cudaFreeAsync(scratch, st);
    if (ce != cudaSuccess) {
        set_error("rz_ingest_json_dev: %s", cudaGetErrorString(ce));
        return RZ_ECUDA;
    }
    if (rc != RZ_OK) return rc;
    return report(herr, error_offset, "rz_ingest_json_dev");
}

int rz_ingest_json(const char* path, size_t capacity, uint8_t* planes, float* policy, float* z, size_t* n_records,
                   size_t* error_offset) {
    RZ_REQUIRE(path && n_records, "rz_ingest_json: null pointer");
    if (error_offset) *error_offset = (size_t)-1;
    FILE* f = fopen(path, "rb");
    if (!f) { set_error("rz_ingest_json: cannot open %s", path); return RZ_EIO; }
    std::string text;
    char buf[1 << 16];
    size_t got;
    while ((got = fread(buf, 1, sizeof(buf), f)) > 0) text.append(buf, got);
    const bool bad = ferror(f) != 0;
    fclose(f);
    if (bad) { set_error("rz_ingest_json: read error on %s", path); return RZ_EIO; }
    const size_t n = text.size();
    char* d = nullptr;
    RZ_CUDA_TRY(cudaMalloc((void**)&d, n + 16));
    cudaError_t ce = n ? cudaMemcpy(d, text.data(), n, cudaMemcpyHostToDevice) : cudaSuccess;
    int rc = RZ_OK;
    size_t nr = 0;
    if (ce == cudaSuccess) rc = rz_ingest_json_dev(d, n, 0, nullptr, nullptr, nullptr, &nr, error_offset, 0);  // the record count
    char* out = nullptr;
    if (ce == cudaSuccess && rc == RZ_ECAPACITY && nr <= capacity && !(planes && policy && z)) {
        set_error("rz_ingest_json: null pointer");
        rc = RZ_EINVAL;
    }
    if (ce == cudaSuccess && rc == RZ_ECAPACITY && nr <= capacity) {
        ce = cudaMalloc((void**)&out, nr * (128 + 256 + sizeof(float)));
        if (ce == cudaSuccess)
            rc = rz_ingest_json_dev(d, n, nr, (uint8_t*)out, (float*)(out + nr * 128), (float*)(out + nr * 384), &nr, error_offset, 0);
    }
    *n_records = nr;
    if (rc == RZ_OK && ce == cudaSuccess && nr) {
        ce = cudaMemcpy(planes, out, nr * 128, cudaMemcpyDeviceToHost);
        if (ce == cudaSuccess) ce = cudaMemcpy(policy, out + nr * 128, nr * 256, cudaMemcpyDeviceToHost);
        if (ce == cudaSuccess) ce = cudaMemcpy(z, out + nr * 384, nr * sizeof(float), cudaMemcpyDeviceToHost);
    }
    cudaFree(out);
    cudaFree(d);
    if (rc != RZ_OK) return rc;
    if (ce != cudaSuccess) { set_error("rz_ingest_json: %s", cudaGetErrorString(ce)); return RZ_ECUDA; }
    return RZ_OK;
}

}  // extern "C"
