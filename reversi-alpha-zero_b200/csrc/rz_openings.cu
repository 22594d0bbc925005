// rz_openings.cu -- every distinct opening of p plies, enumerated on the device (rz_openings_enumerate); the opening
// book's graph over them (rz_openings_book_graph) and the children of any list of book nodes (rz_openings_book_children).
//
// Level by level from the initial position: each frontier position is expanded to its children (rz_openings.cuh), the
// children are sorted by their canonical key (two stable CUB radix sorts, low word then high word, so that equal keys
// stay in child order), and the first child of every key -- the one with the least (parent index, move square) -- becomes
// the class's representative, in the orientation its own moves reach.  The representatives, in ascending key order, are
// the next frontier.  Every step is a scan, a stable sort or a gather: the output does not depend on the schedule.
#include <climits>
#include <cub/cub.cuh>
#include <vector>

#include "rz_common.cuh"
#include "rz_openings.cuh"

namespace rz {
namespace openings {

constexpr int kThreads = 256;

inline unsigned blocks_for(size_t n) { return (unsigned)((n + kThreads - 1) / kThreads); }

__global__ void __launch_bounds__(kThreads) count_kernel(const u64* __restrict__ own, const u64* __restrict__ enemy, size_t n,
                                                         uint64_t* __restrict__ count) {
    const size_t i = (size_t)blockIdx.x * kThreads + threadIdx.x;
    if (i < n) count[i] = (uint64_t)popc64(kept_moves(own[i], enemy[i]));
}

// children of parent i at offset[i] .. : canonical key, the child's index (the sort's value) and parent * 64 + square
__global__ void __launch_bounds__(kThreads) expand_kernel(const u64* __restrict__ own, const u64* __restrict__ enemy, size_t n,
                                                          const uint64_t* __restrict__ offset, u64* __restrict__ k_hi,
                                                          u64* __restrict__ k_lo, uint32_t* __restrict__ index,
                                                          u64* __restrict__ origin) {
    const size_t i = (size_t)blockIdx.x * kThreads + threadIdx.x;
    if (i >= n) return;
    const u64 o = own[i], e = enemy[i];
    size_t c = offset[i];
    for (u64 m = find_correct_moves(o, e); m; m &= m - 1) {
        const int sq = ctz64(m);
        u64 co, ce;
        if (!child(o, e, sq, co, ce)) continue;
        canonical(co, ce, k_hi[c], k_lo[c]);
        index[c] = (uint32_t)c;
        origin[c] = (u64)i * 64 + (u64)sq;
        ++c;
    }
}

__global__ void __launch_bounds__(kThreads) gather_kernel(const u64* __restrict__ src, const uint32_t* __restrict__ index, size_t n,
                                                          u64* __restrict__ dst) {
    const size_t j = (size_t)blockIdx.x * kThreads + threadIdx.x;
    if (j < n) dst[j] = src[index[j]];
}

// head[j] = 1 where the sorted key j differs from key j - 1 (k_hi sorted, k_lo in child order)
__global__ void __launch_bounds__(kThreads) head_kernel(const u64* __restrict__ hi_sorted, const u64* __restrict__ k_lo,
                                                        const uint32_t* __restrict__ index, size_t n, uint8_t* __restrict__ head) {
    const size_t j = (size_t)blockIdx.x * kThreads + threadIdx.x;
    if (j >= n) return;
    head[j] = j == 0 || hi_sorted[j] != hi_sorted[j - 1] || k_lo[index[j]] != k_lo[index[j - 1]];
}

// next frontier: representative k is child rep[k]; its position and moves (its parent's moves, then its square)
__global__ void __launch_bounds__(kThreads) next_kernel(const u64* __restrict__ own, const u64* __restrict__ enemy,
                                                        const uint8_t* __restrict__ moves, int level, int stride,
                                                        const uint32_t* __restrict__ rep, const u64* __restrict__ origin, size_t n,
                                                        u64* __restrict__ own_out, u64* __restrict__ enemy_out,
                                                        uint8_t* __restrict__ moves_out) {
    const size_t k = (size_t)blockIdx.x * kThreads + threadIdx.x;
    if (k >= n) return;
    const u64 org = origin[rep[k]];
    const size_t parent = (size_t)(org >> 6);
    const int sq = (int)(org & 63);
    u64 co, ce;
    child(own[parent], enemy[parent], sq, co, ce);
    own_out[k] = co;
    enemy_out[k] = ce;
    if (!moves_out) return;   // the book graph keeps no move sequences
    for (int j = 0; j < level; ++j) moves_out[k * stride + j] = moves[parent * stride + j];
    moves_out[k * stride + level] = (uint8_t)sq;
}

// canonical keys of n positions (the book graph's binary-search tables)
__global__ void __launch_bounds__(kThreads) key_kernel(const u64* __restrict__ own, const u64* __restrict__ enemy, size_t n,
                                                       u64* __restrict__ k_hi, u64* __restrict__ k_lo) {
    const size_t i = (size_t)blockIdx.x * kThreads + threadIdx.x;
    if (i < n) canonical(own[i], enemy[i], k_hi[i], k_lo[i]);
}

// legal moves of n positions: the book graph's edge counts
__global__ void __launch_bounds__(kThreads) legal_count_kernel(const u64* __restrict__ own, const u64* __restrict__ enemy, size_t n,
                                                               uint64_t* __restrict__ count) {
    const size_t i = (size_t)blockIdx.x * kThreads + threadIdx.x;
    if (i < n) count[i] = (uint64_t)popc64(find_correct_moves(own[i], enemy[i]));
}

// the edges of n nodes of one level, at their CSR offsets, against the next level's n_next keys
__global__ void __launch_bounds__(kThreads) edge_kernel(const u64* __restrict__ own, const u64* __restrict__ enemy, size_t n,
                                                        const uint64_t* __restrict__ offset, const u64* __restrict__ next_hi,
                                                        const u64* __restrict__ next_lo, size_t n_next, uint8_t* __restrict__ square,
                                                        int32_t* __restrict__ child_index) {
    const size_t i = (size_t)blockIdx.x * kThreads + threadIdx.x;
    if (i >= n) return;
    book_edges(own[i], enemy[i], next_hi, next_lo, n_next, square + offset[i], child_index + offset[i]);
}

// the children of n nodes at their CSR offsets, against a sorted level's n_next keys
__global__ void __launch_bounds__(kThreads) children_kernel(const u64* __restrict__ own, const u64* __restrict__ enemy, size_t n,
                                                            const uint64_t* __restrict__ offset, const u64* __restrict__ next_hi,
                                                            const u64* __restrict__ next_lo, size_t n_next,
                                                            uint8_t* __restrict__ square, int32_t* __restrict__ child_index,
                                                            u64* __restrict__ c_own, u64* __restrict__ c_enemy, u64* __restrict__ c_hi,
                                                            u64* __restrict__ c_lo, uint8_t* __restrict__ kind) {
    const size_t i = (size_t)blockIdx.x * kThreads + threadIdx.x;
    if (i >= n) return;
    const size_t o = offset[i];
    book_children(own[i], enemy[i], next_hi, next_lo, n_next, square + o, child_index + o, c_own + o, c_enemy + o, c_hi + o,
                  c_lo + o, kind + o);
}

// device buffers of one call, freed on every return
struct Buffers {
    const char* who;
    std::vector<void*> held;
    explicit Buffers(const char* who_) : who(who_) {}
    ~Buffers() { for (void* p : held) cudaFree(p); }
    template <typename T>
    int get(T** out, size_t count) {
        void* p = nullptr;
        const size_t bytes = count ? count * sizeof(T) : 1;
        if (cudaMalloc(&p, bytes) != cudaSuccess) {
            cudaGetLastError();
            set_error("%s: cudaMalloc(%zu bytes) failed", who, bytes);
            return RZ_ENOMEM;
        }
        held.push_back(p);
        *out = (T*)p;
        return RZ_OK;
    }
    void release(void* p) {
        for (size_t i = 0; i < held.size(); ++i)
            if (held[i] == p) { cudaFree(p); held.erase(held.begin() + (long)i); return; }
    }
};

// level 0: the initial position, black to move, in buffers of buf
int start_level(Buffers& buf, cudaStream_t st, u64** own, u64** enemy) {
    RZ_TRY(buf.get(own, 1));
    RZ_TRY(buf.get(enemy, 1));
    const u64 start[2] = {kStartBlack, kStartWhite};
    RZ_CUDA_TRY(cudaMemcpyAsync(*own, &start[0], sizeof(u64), cudaMemcpyHostToDevice, st));
    RZ_CUDA_TRY(cudaMemcpyAsync(*enemy, &start[1], sizeof(u64), cudaMemcpyHostToDevice, st));
    return RZ_OK;
}

// One level: the n positions (own, enemy) of `level` plies -> the next level's representatives in ascending key order,
// in new buffers of buf (*own_next, *enemy_next, *n_next).  With moves (n x stride, `level` squares each) the next
// level's moves go to *moves_next; moves = NULL keeps none.  The input buffers stay the caller's.
int expand_level(Buffers& buf, cudaStream_t st, const u64* own, const u64* enemy, const uint8_t* moves, int level, int stride,
                 size_t n, u64** own_next, u64** enemy_next, uint8_t** moves_next, size_t* n_next) {
    uint64_t *count, *offset;
    RZ_TRY(buf.get(&count, n + 1));
    RZ_TRY(buf.get(&offset, n + 1));
    count_kernel<<<blocks_for(n), kThreads, 0, st>>>(own, enemy, n, count);
    RZ_LAUNCH_CHECK();
    RZ_CUDA_TRY(cudaMemsetAsync(count + n, 0, sizeof(uint64_t), st));
    size_t tmp_bytes = 0;
    RZ_CUDA_TRY(cub::DeviceScan::ExclusiveSum(nullptr, tmp_bytes, count, offset, (int64_t)(n + 1), st));
    void* tmp;
    RZ_TRY(buf.get((uint8_t**)&tmp, tmp_bytes));
    RZ_CUDA_TRY(cub::DeviceScan::ExclusiveSum(tmp, tmp_bytes, count, offset, (int64_t)(n + 1), st));
    uint64_t m = 0;
    RZ_CUDA_TRY(cudaMemcpyAsync(&m, offset + n, sizeof(uint64_t), cudaMemcpyDeviceToHost, st));
    RZ_CUDA_TRY(cudaStreamSynchronize(st));
    buf.release(tmp);
    buf.release(count);
    if (m > (uint64_t)INT_MAX) {
        set_error("%s: %llu children at ply %d exceed the sort's %d items", buf.who, (unsigned long long)m, level + 1, INT_MAX);
        return RZ_ENOMEM;
    }
    u64 *k_hi, *k_lo, *origin, *sorted_a, *sorted_b;
    uint32_t *index, *index_a, *index_b;
    RZ_TRY(buf.get(&k_hi, m));
    RZ_TRY(buf.get(&k_lo, m));
    RZ_TRY(buf.get(&origin, m));
    RZ_TRY(buf.get(&index, m));
    expand_kernel<<<blocks_for(n), kThreads, 0, st>>>(own, enemy, n, offset, k_hi, k_lo, index, origin);
    RZ_LAUNCH_CHECK();
    RZ_TRY(buf.get(&sorted_a, m));
    RZ_TRY(buf.get(&sorted_b, m));
    RZ_TRY(buf.get(&index_a, m));
    RZ_TRY(buf.get(&index_b, m));
    // low word first, then high word: radix sort is stable, so this orders by (hi, lo) and keeps child order in a class
    tmp_bytes = 0;
    RZ_CUDA_TRY(cub::DeviceRadixSort::SortPairs(nullptr, tmp_bytes, k_lo, sorted_a, index, index_a, (int)m, 0, 64, st));
    RZ_TRY(buf.get((uint8_t**)&tmp, tmp_bytes));
    RZ_CUDA_TRY(cub::DeviceRadixSort::SortPairs(tmp, tmp_bytes, k_lo, sorted_a, index, index_a, (int)m, 0, 64, st));
    gather_kernel<<<blocks_for(m), kThreads, 0, st>>>(k_hi, index_a, m, sorted_b);
    RZ_LAUNCH_CHECK();
    RZ_CUDA_TRY(cub::DeviceRadixSort::SortPairs(tmp, tmp_bytes, sorted_b, sorted_a, index_a, index_b, (int)m, 0, 64, st));
    buf.release(tmp);
    uint8_t* head;
    RZ_TRY(buf.get(&head, m));
    head_kernel<<<blocks_for(m), kThreads, 0, st>>>(sorted_a, k_lo, index_b, m, head);
    RZ_LAUNCH_CHECK();
    int* n_sel;
    RZ_TRY(buf.get(&n_sel, 1));
    tmp_bytes = 0;
    RZ_CUDA_TRY(cub::DeviceSelect::Flagged(nullptr, tmp_bytes, index_b, head, index_a, n_sel, (int)m, st));
    RZ_TRY(buf.get((uint8_t**)&tmp, tmp_bytes));
    RZ_CUDA_TRY(cub::DeviceSelect::Flagged(tmp, tmp_bytes, index_b, head, index_a, n_sel, (int)m, st));
    int n_sel_host = 0;
    RZ_CUDA_TRY(cudaMemcpyAsync(&n_sel_host, n_sel, sizeof(int), cudaMemcpyDeviceToHost, st));
    RZ_CUDA_TRY(cudaStreamSynchronize(st));
    for (void* p : {(void*)tmp, (void*)head, (void*)n_sel, (void*)k_hi, (void*)sorted_a, (void*)sorted_b, (void*)index,
                    (void*)index_b, (void*)offset})
        buf.release(p);
    uint8_t* moves2 = nullptr;
    RZ_TRY(buf.get(own_next, (size_t)n_sel_host));
    RZ_TRY(buf.get(enemy_next, (size_t)n_sel_host));
    if (moves) RZ_TRY(buf.get(&moves2, (size_t)n_sel_host * stride));
    next_kernel<<<blocks_for((size_t)n_sel_host), kThreads, 0, st>>>(own, enemy, moves, level, stride, index_a, origin,
                                                                     (size_t)n_sel_host, *own_next, *enemy_next, moves2);
    RZ_LAUNCH_CHECK();
    RZ_CUDA_TRY(cudaStreamSynchronize(st));
    for (void* p : {(void*)index_a, (void*)origin, (void*)k_lo}) buf.release(p);
    if (moves_next) *moves_next = moves2;
    *n_next = (size_t)n_sel_host;
    return RZ_OK;
}

}  // namespace openings
}  // namespace rz

using namespace rz;
using namespace rz::openings;

extern "C" int rz_openings_enumerate(int plies, uint64_t* own_out, uint64_t* enemy_out, uint8_t* moves_out, size_t cap,
                                     size_t* n_out, uint64_t* level_counts) {
    RZ_REQUIRE(plies >= 1 && plies <= 12, "rz_openings_enumerate: plies = %d outside 1..12", plies);
    RZ_REQUIRE(n_out, "rz_openings_enumerate: null n_out");
    RZ_REQUIRE(cap == 0 || (own_out && enemy_out && moves_out), "rz_openings_enumerate: null output with cap = %zu", cap);
    *n_out = 0;
    const cudaStream_t st = 0;
    Buffers buf("rz_openings_enumerate");
    // the frontier: level 0 is the initial position, black to move
    u64 *own, *enemy;
    uint8_t* moves;
    size_t n = 1;
    RZ_TRY(start_level(buf, st, &own, &enemy));
    RZ_TRY(buf.get(&moves, (size_t)plies));
    if (level_counts) level_counts[0] = 1;
    for (int level = 0; level < plies; ++level) {
        u64 *own2, *enemy2;
        uint8_t* moves2;
        RZ_TRY(expand_level(buf, st, own, enemy, moves, level, plies, n, &own2, &enemy2, &moves2, &n));
        for (void* p : {(void*)own, (void*)enemy, (void*)moves}) buf.release(p);
        own = own2; enemy = enemy2; moves = moves2;
        if (level_counts) level_counts[level + 1] = n;
    }
    *n_out = n;
    if (cap == 0) return RZ_OK;
    if (cap < n) {
        set_error("rz_openings_enumerate: %zu openings of %d plies, room for %zu", n, plies, cap);
        return RZ_ECAPACITY;
    }
    RZ_CUDA_TRY(cudaMemcpy(own_out, own, n * sizeof(u64), cudaMemcpyDeviceToHost));
    RZ_CUDA_TRY(cudaMemcpy(enemy_out, enemy, n * sizeof(u64), cudaMemcpyDeviceToHost));
    RZ_CUDA_TRY(cudaMemcpy(moves_out, moves, n * (size_t)plies, cudaMemcpyDeviceToHost));
    return RZ_OK;
}

// The book graph: levels 0 .. plies as rz_openings_enumerate builds them (no move sequences), kept side by side in one
// node array; then per node its canonical key, its legal-move count and an exclusive scan of the counts (the CSR
// offsets, last level 0), and per level below the last the edge kernel against the next level's keys.
extern "C" int rz_openings_book_graph(int plies, uint64_t* own_out, uint64_t* enemy_out, uint64_t* key_hi_out,
                                      uint64_t* key_lo_out, size_t cap_nodes, size_t* n_nodes,
                                      uint64_t* level_counts, uint64_t* edge_offset, uint8_t* edge_square,
                                      int32_t* edge_child, size_t cap_edges, size_t* n_edges) {
    RZ_REQUIRE(plies >= 1 && plies <= 10, "rz_openings_book_graph: plies = %d outside 1..10", plies);
    RZ_REQUIRE(n_nodes && n_edges, "rz_openings_book_graph: null n_nodes or n_edges");
    RZ_REQUIRE(cap_nodes == 0 || (own_out && enemy_out && edge_offset && (cap_edges == 0 || (edge_square && edge_child))),
               "rz_openings_book_graph: null output with cap_nodes = %zu", cap_nodes);
    *n_nodes = 0;
    *n_edges = 0;
    const cudaStream_t st = 0;
    Buffers buf("rz_openings_book_graph");
    std::vector<u64*> lv_own(plies + 1), lv_enemy(plies + 1);
    std::vector<size_t> count(plies + 1), first(plies + 2, 0);
    RZ_TRY(start_level(buf, st, &lv_own[0], &lv_enemy[0]));
    count[0] = 1;
    for (int level = 0; level < plies; ++level)
        RZ_TRY(expand_level(buf, st, lv_own[level], lv_enemy[level], nullptr, level, 0, count[level], &lv_own[level + 1],
                            &lv_enemy[level + 1], nullptr, &count[level + 1]));
    for (int level = 0; level <= plies; ++level) first[level + 1] = first[level] + count[level];
    const size_t n = first[plies + 1], n_inner = first[plies];
    u64 *own, *enemy, *k_hi, *k_lo;
    uint64_t *moves, *offset;
    RZ_TRY(buf.get(&own, n));
    RZ_TRY(buf.get(&enemy, n));
    for (int level = 0; level <= plies; ++level) {
        RZ_CUDA_TRY(cudaMemcpyAsync(own + first[level], lv_own[level], count[level] * sizeof(u64), cudaMemcpyDeviceToDevice, st));
        RZ_CUDA_TRY(cudaMemcpyAsync(enemy + first[level], lv_enemy[level], count[level] * sizeof(u64), cudaMemcpyDeviceToDevice, st));
    }
    RZ_CUDA_TRY(cudaStreamSynchronize(st));
    for (int level = 0; level <= plies; ++level) { buf.release(lv_own[level]); buf.release(lv_enemy[level]); }
    RZ_TRY(buf.get(&k_hi, n));
    RZ_TRY(buf.get(&k_lo, n));
    RZ_TRY(buf.get(&moves, n + 1));
    RZ_TRY(buf.get(&offset, n + 1));
    key_kernel<<<blocks_for(n), kThreads, 0, st>>>(own, enemy, n, k_hi, k_lo);
    RZ_LAUNCH_CHECK();
    legal_count_kernel<<<blocks_for(n_inner), kThreads, 0, st>>>(own, enemy, n_inner, moves);
    RZ_LAUNCH_CHECK();
    RZ_CUDA_TRY(cudaMemsetAsync(moves + n_inner, 0, (n + 1 - n_inner) * sizeof(uint64_t), st));
    size_t tmp_bytes = 0;
    RZ_CUDA_TRY(cub::DeviceScan::ExclusiveSum(nullptr, tmp_bytes, moves, offset, (int64_t)(n + 1), st));
    uint8_t* tmp;
    RZ_TRY(buf.get(&tmp, tmp_bytes));
    RZ_CUDA_TRY(cub::DeviceScan::ExclusiveSum(tmp, tmp_bytes, moves, offset, (int64_t)(n + 1), st));
    uint64_t m = 0;
    RZ_CUDA_TRY(cudaMemcpyAsync(&m, offset + n, sizeof(uint64_t), cudaMemcpyDeviceToHost, st));
    RZ_CUDA_TRY(cudaStreamSynchronize(st));
    buf.release(tmp);
    buf.release(moves);
    uint8_t* square;
    int32_t* child_index;
    RZ_TRY(buf.get(&square, m));
    RZ_TRY(buf.get(&child_index, m));
    for (int level = 0; level < plies; ++level) {
        edge_kernel<<<blocks_for(count[level]), kThreads, 0, st>>>(own + first[level], enemy + first[level], count[level],
                                                                   offset + first[level], k_hi + first[level + 1],
                                                                   k_lo + first[level + 1], count[level + 1], square, child_index);
        RZ_LAUNCH_CHECK();
    }
    RZ_CUDA_TRY(cudaStreamSynchronize(st));
    *n_nodes = n;
    *n_edges = (size_t)m;
    if (level_counts)
        for (int level = 0; level <= plies; ++level) level_counts[level] = count[level];
    if (cap_nodes == 0) return RZ_OK;
    if (cap_nodes < n || cap_edges < m) {
        set_error("rz_openings_book_graph: %zu nodes and %llu edges of %d plies, room for %zu and %zu", n,
                  (unsigned long long)m, plies, cap_nodes, cap_edges);
        return RZ_ECAPACITY;
    }
    RZ_CUDA_TRY(cudaMemcpy(own_out, own, n * sizeof(u64), cudaMemcpyDeviceToHost));
    RZ_CUDA_TRY(cudaMemcpy(enemy_out, enemy, n * sizeof(u64), cudaMemcpyDeviceToHost));
    if (key_hi_out) RZ_CUDA_TRY(cudaMemcpy(key_hi_out, k_hi, n * sizeof(u64), cudaMemcpyDeviceToHost));
    if (key_lo_out) RZ_CUDA_TRY(cudaMemcpy(key_lo_out, k_lo, n * sizeof(u64), cudaMemcpyDeviceToHost));
    RZ_CUDA_TRY(cudaMemcpy(edge_offset, offset, (n + 1) * sizeof(uint64_t), cudaMemcpyDeviceToHost));
    RZ_CUDA_TRY(cudaMemcpy(edge_square, square, (size_t)m, cudaMemcpyDeviceToHost));
    RZ_CUDA_TRY(cudaMemcpy(edge_child, child_index, (size_t)m * sizeof(int32_t), cudaMemcpyDeviceToHost));
    return RZ_OK;
}

// The children of any n nodes: the nodes and the level's keys copied to the device, the legal-move counts, an exclusive
// scan of them (the CSR offsets), and the children kernel, one node per thread.
extern "C" int rz_openings_book_children(const uint64_t* own_in, const uint64_t* enemy_in, size_t n, const uint64_t* next_hi_in,
                                         const uint64_t* next_lo_in, size_t n_next, uint64_t* edge_offset, uint8_t* edge_square,
                                         int32_t* edge_child, uint64_t* child_own, uint64_t* child_enemy, uint64_t* child_hi,
                                         uint64_t* child_lo, uint8_t* child_kind, size_t cap_edges, size_t* n_edges) {
    RZ_REQUIRE(n_edges, "rz_openings_book_children: null n_edges");
    RZ_REQUIRE(n == 0 || (own_in && enemy_in), "rz_openings_book_children: null nodes with n = %zu", n);
    RZ_REQUIRE(n_next == 0 || (next_hi_in && next_lo_in), "rz_openings_book_children: null keys with n_next = %zu", n_next);
    RZ_REQUIRE(!edge_offset || (edge_square && edge_child && child_own && child_enemy && child_hi && child_lo && child_kind),
               "rz_openings_book_children: edge_offset without the other outputs");
    *n_edges = 0;
    if (n == 0) {
        if (edge_offset) edge_offset[0] = 0;
        return RZ_OK;
    }
    const cudaStream_t st = 0;
    Buffers buf("rz_openings_book_children");
    u64 *own, *enemy, *next_hi, *next_lo;
    uint64_t *count, *offset;
    RZ_TRY(buf.get(&own, n));
    RZ_TRY(buf.get(&enemy, n));
    RZ_TRY(buf.get(&next_hi, n_next));
    RZ_TRY(buf.get(&next_lo, n_next));
    RZ_TRY(buf.get(&count, n + 1));
    RZ_TRY(buf.get(&offset, n + 1));
    RZ_CUDA_TRY(cudaMemcpyAsync(own, own_in, n * sizeof(u64), cudaMemcpyHostToDevice, st));
    RZ_CUDA_TRY(cudaMemcpyAsync(enemy, enemy_in, n * sizeof(u64), cudaMemcpyHostToDevice, st));
    if (n_next) {
        RZ_CUDA_TRY(cudaMemcpyAsync(next_hi, next_hi_in, n_next * sizeof(u64), cudaMemcpyHostToDevice, st));
        RZ_CUDA_TRY(cudaMemcpyAsync(next_lo, next_lo_in, n_next * sizeof(u64), cudaMemcpyHostToDevice, st));
    }
    legal_count_kernel<<<blocks_for(n), kThreads, 0, st>>>(own, enemy, n, count);
    RZ_LAUNCH_CHECK();
    RZ_CUDA_TRY(cudaMemsetAsync(count + n, 0, sizeof(uint64_t), st));
    size_t tmp_bytes = 0;
    RZ_CUDA_TRY(cub::DeviceScan::ExclusiveSum(nullptr, tmp_bytes, count, offset, (int64_t)(n + 1), st));
    uint8_t* tmp;
    RZ_TRY(buf.get(&tmp, tmp_bytes));
    RZ_CUDA_TRY(cub::DeviceScan::ExclusiveSum(tmp, tmp_bytes, count, offset, (int64_t)(n + 1), st));
    uint64_t m = 0;
    RZ_CUDA_TRY(cudaMemcpyAsync(&m, offset + n, sizeof(uint64_t), cudaMemcpyDeviceToHost, st));
    RZ_CUDA_TRY(cudaStreamSynchronize(st));
    *n_edges = (size_t)m;
    if (!edge_offset) return RZ_OK;
    if (cap_edges < m) {
        set_error("rz_openings_book_children: %llu children of %zu nodes, room for %zu", (unsigned long long)m, n, cap_edges);
        return RZ_ECAPACITY;
    }
    buf.release(tmp);
    buf.release(count);
    uint8_t *square, *kind;
    int32_t* child_index;
    u64 *c_own, *c_enemy, *c_hi, *c_lo;
    RZ_TRY(buf.get(&square, m));
    RZ_TRY(buf.get(&kind, m));
    RZ_TRY(buf.get(&child_index, m));
    RZ_TRY(buf.get(&c_own, m));
    RZ_TRY(buf.get(&c_enemy, m));
    RZ_TRY(buf.get(&c_hi, m));
    RZ_TRY(buf.get(&c_lo, m));
    children_kernel<<<blocks_for(n), kThreads, 0, st>>>(own, enemy, n, offset, next_hi, next_lo, n_next, square, child_index, c_own,
                                                        c_enemy, c_hi, c_lo, kind);
    RZ_LAUNCH_CHECK();
    RZ_CUDA_TRY(cudaMemcpy(edge_offset, offset, (n + 1) * sizeof(uint64_t), cudaMemcpyDeviceToHost));
    RZ_CUDA_TRY(cudaMemcpy(edge_square, square, (size_t)m, cudaMemcpyDeviceToHost));
    RZ_CUDA_TRY(cudaMemcpy(edge_child, child_index, (size_t)m * sizeof(int32_t), cudaMemcpyDeviceToHost));
    RZ_CUDA_TRY(cudaMemcpy(child_own, c_own, (size_t)m * sizeof(u64), cudaMemcpyDeviceToHost));
    RZ_CUDA_TRY(cudaMemcpy(child_enemy, c_enemy, (size_t)m * sizeof(u64), cudaMemcpyDeviceToHost));
    RZ_CUDA_TRY(cudaMemcpy(child_hi, c_hi, (size_t)m * sizeof(u64), cudaMemcpyDeviceToHost));
    RZ_CUDA_TRY(cudaMemcpy(child_lo, c_lo, (size_t)m * sizeof(u64), cudaMemcpyDeviceToHost));
    RZ_CUDA_TRY(cudaMemcpy(child_kind, kind, (size_t)m, cudaMemcpyDeviceToHost));
    return RZ_OK;
}
