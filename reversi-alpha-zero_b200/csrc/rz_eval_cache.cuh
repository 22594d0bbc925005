// rz_eval_cache.cuh -- device-side evaluation cache of the self-play engine (included by rz_engine.cu).
//
// The tower is a pure function of its input board: every output row goes through the same operations whichever batch row
// the board lands in.  So a leaf whose dihedral-transformed (own, enemy) was evaluated before can take that policy / value
// instead of a tower row, and the search sees the same bits.  All games start from one position, so early leaves repeat
// across games.
//
// Table: n_sets x kCacheWays entries of 288 B in HBM, keyed by the transformed board, tagged with the network's weights
// version (rz_net::weights_version), so loading new weights makes every older entry a miss.  An insert overwrites the
// set's oldest entry (a FIFO counter per set).
//
// Concurrency: the two slot groups share the table and their streams are not ordered against each other, so a group's
// lookups can run while the other group's insert kernel writes.  Each entry carries a sequence word that is odd while a
// writer fills it: a writer claims the entry by a compare-and-swap to odd, writes, and publishes the next even value; a
// reader takes the data only when it saw the same even sequence word before and after copying it, with the right key and
// weights version.  A reader that loses such a race treats the leaf as a miss, which costs one tower row and changes
// no result.  Hit counts of a two-group engine therefore depend on timing; the games do not.
#pragma once

constexpr int kCacheWays = 8;

struct __align__(16) EvalCacheEntry {
    u64 own, enemy;    // transformed board, side to move first
    uint32_t seq;      // odd while a writer fills the entry
    uint32_t gen;      // weights version of the network that computed it (0: empty)
    float value;
    uint32_t pad;
    float policy[64];  // in the transformed frame, as the tower wrote it
};
static_assert(sizeof(EvalCacheEntry) == 288, "cache entry layout");

struct EvalCache {
    EvalCacheEntry* entries;  // [n_sets][kCacheWays]
    uint32_t* next;           // [n_sets] FIFO insert counter
    uint32_t n_sets;          // 0: the cache is off
    uint32_t gen;             // current weights version
};

__device__ __forceinline__ EvalCacheEntry* cache_set(const EvalCache& t, u64 own, u64 enemy) {
    return t.entries + (size_t)(hash_key(own, enemy, 0) % t.n_sets) * kCacheWays;
}

__device__ __forceinline__ uint32_t volatile_load(const uint32_t* p) { return *(const volatile uint32_t*)p; }

// One thread: copies the cached result of (own, enemy) to policy_out[64] / *value_out and returns true, or returns false
// (policy_out may then hold a partial copy).
__device__ bool cache_lookup(const EvalCache& t, u64 own, u64 enemy, float* policy_out, float* value_out) {
    EvalCacheEntry* set = cache_set(t, own, enemy);
    int way = -1;
#pragma unroll
    for (int w = 0; w < kCacheWays; ++w) {
        const ulonglong2 k = __ldcg(reinterpret_cast<const ulonglong2*>(set + w));
        const uint2 m = __ldcg(reinterpret_cast<const uint2*>(&set[w].seq));
        if (k.x == own && k.y == enemy && m.y == t.gen && !(m.x & 1u)) way = w;
    }
    if (way < 0) return false;
    EvalCacheEntry* e = set + way;
    const uint32_t s1 = volatile_load(&e->seq);
    __threadfence();
    const ulonglong2 k = __ldcg(reinterpret_cast<const ulonglong2*>(e));
    const uint32_t g = __ldcg(&e->gen);
    const float v = __ldcg(&e->value);
    const float4* src = reinterpret_cast<const float4*>(e->policy);
    float4* dst = reinterpret_cast<float4*>(policy_out);
#pragma unroll
    for (int i = 0; i < 16; ++i) dst[i] = __ldcg(src + i);
    __threadfence();
    const uint32_t s2 = volatile_load(&e->seq);
    if (s1 != s2 || (s1 & 1u) || k.x != own || k.y != enemy || g != t.gen) return false;
    *value_out = v;
    return true;
}

// After the tower: rows [0, *count) of the group's batch into the table, one thread per row.  A row whose key is already
// present (another leaf of the same wave, or of the other group, sent the same board to the tower) is counted in *repeats
// and not stored again.
__global__ void cache_insert_kernel(const EvalCache t, const u64* __restrict__ own, const u64* __restrict__ enemy,
                                    const float* __restrict__ policy, const float* __restrict__ value,
                                    const uint32_t* __restrict__ count, unsigned long long* repeats) {
    const uint32_t n = *count;
    for (uint32_t r = blockIdx.x * blockDim.x + threadIdx.x; r < n; r += gridDim.x * blockDim.x) {
        const u64 o = own[r], en = enemy[r];
        EvalCacheEntry* set = cache_set(t, o, en);
        bool present = false;
#pragma unroll
        for (int w = 0; w < kCacheWays; ++w) {
            const ulonglong2 k = __ldcg(reinterpret_cast<const ulonglong2*>(set + w));
            const uint32_t g = __ldcg(&set[w].gen);
            if (k.x == o && k.y == en && g == t.gen) present = true;
        }
        const unsigned rep = __ballot_sync(__activemask(), present);
        if (present) {
            if ((threadIdx.x & 31) == (unsigned)(__ffs(rep) - 1)) atomicAdd(repeats, (unsigned long long)__popc(rep));
            continue;
        }
        EvalCacheEntry* e = set + atomicAdd(t.next + (set - t.entries) / kCacheWays, 1u) % kCacheWays;
        const uint32_t s = volatile_load(&e->seq);
        if ((s & 1u) || atomicCAS(&e->seq, s, s + 1u) != s) continue;  // another writer holds the entry: drop this insert
        __threadfence();
        e->own = o; e->enemy = en; e->gen = t.gen; e->value = value[r];
        const float4* src = reinterpret_cast<const float4*>(policy + (size_t)r * 64);
        float4* dst = reinterpret_cast<float4*>(e->policy);
#pragma unroll
        for (int i = 0; i < 16; ++i) dst[i] = src[i];
        __threadfence();
        atomicExch(&e->seq, s + 2u);
    }
}
