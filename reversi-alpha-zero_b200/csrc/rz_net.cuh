// rz_net.cuh -- policy/value network object shared by the inference kernels and the engine.
//
// Architecture = the reference's ReversiModel.build (agent/model.py:28-72): conv3x3(2->F)+BN+ReLU,
// R residual blocks of two conv3x3(F->F)+BN (ReLU after the first, skip-add then ReLU after the
// second), policy head conv1x1(F->2)+BN+ReLU -> Dense(128->64, softmax), value head
// conv1x1(F->1)+BN+ReLU -> Dense(64->V, relu) -> Dense(V->1, tanh).  BN is folded at load time into a
// per-channel fp32 (scale, shift) applied in the conv epilogue:
//   scale = gamma / sqrt(var + 1e-3),  shift = beta + (bias - mean) * scale.
#pragma once
#include <cuda_fp16.h>
#include <mutex>
#include "rz_common.cuh"

struct rz_net {
    rz_net_cfg cfg;
    int device;
    bool loaded;
    uint64_t weights_version;  // 1, 2, ...: counts the weight loads (tags the engine's evaluation cache entries)
    size_t blob_floats;
    float* blob;         // device copy of the fp32 blob (Keras layouts), used by the generic kernel and the heads
    float* scale_shift;  // [n_conv_layers][2][F] folded BN of conv0 + tower convs; then heads: [2][2] policy, [2][1] value
    // offsets (in floats) into blob
    size_t off_conv0, off_res0, res_stride_conv;  // kernel offset of conv0; of res0.conv1; floats per (conv+bn) group
    size_t off_policy_conv, off_policy_fc_k, off_policy_fc_b;
    size_t off_value_conv, off_value_fc1_k, off_value_fc1_b, off_value_fc2_k, off_value_fc2_b;
    // wgmma tower (F == 64, 128 or 256)
    __half* tc_w0;       // [4 kc][F n][8] fp16: layer-0 weights, K = 18 padded to 32, K-major no-swizzle image
    __half* tc_w;        // F = 256: [2R layers][36 stages][8 kc][256 n][8] fp16, one 32 KB shared-memory image per pipeline stage;
                         // F = 64 / 128: [2R layers][9 taps][F/8 kc][F n][8] fp16, a stage is 3 / 1 consecutive taps
    // fp32 residual-stream scratch of the tower kernel ([CTA][kTowerResFloatsPerCta]); launches from different streams
    // are ordered through res_done, recorded after every launch that uses it
    float* res;
    cudaEvent_t res_done;
    // head features of the wgmma towers ([feat_rows][kHeadFeatures] fp32), grown on demand to a launch's batch capacity;
    // shared by the launches of all streams like res, so ordered through res_done too
    float* feat;
    size_t feat_rows;
    // scratch for the host-buffer predict path
    void* scratch;
    size_t scratch_bytes;
};

namespace rz {

constexpr size_t kTowerResFloatsPerCta = 256 * 128;  // 128 KB: 256 math threads x 128 fp32 accumulators
constexpr int kHeadFeatures = 192;                   // per board: policy head conv (2 x 64, Flatten order c*64 + pix), value (64)

inline int n_conv_layers(const rz_net_cfg& c) { return 1 + 2 * c.res_blocks; }
// per-layer folded BN parameters: scale at [l][0][*], shift at [l][1][*]
inline size_t ss_floats(const rz_net_cfg& c) { return (size_t)n_conv_layers(c) * 2 * c.filters + 4 + 2; }

int net_forward_generic(rz_net* net, const uint64_t* own, const uint64_t* enemy, float* policy, float* value, size_t n,
                        cudaStream_t stream, const uint32_t* n_dev = nullptr);
// batch size known only on the device (count_dev), at most max_n
int net_forward_counted(rz_net* net, const uint64_t* own, const uint64_t* enemy, float* policy, float* value,
                        const uint32_t* count_dev, size_t max_n, int impl, cudaStream_t stream);
// the wgmma tower for F = 256 (rz_net_tc.cu) and, through net_forward_tc_narrow, F = 64 and 128
int net_forward_tc(rz_net* net, const uint64_t* own, const uint64_t* enemy, float* policy, float* value, size_t n,
                   cudaStream_t stream, float* dbg_tower /* nullable: [n][64][F] fp32 tower output */,
                   const uint32_t* n_dev = nullptr /* nullable: actual batch size in device memory (<= n) */,
                   float* dbg_logits = nullptr /* nullable: [n][64] policy logits */, float* dbg_vlogit = nullptr /* nullable: [n] */);
// same function as net_forward_tc, bit for bit, one 8-CTA cluster per 2-board tile (small batches, rz_net_split.cu)
int net_forward_split(rz_net* net, const uint64_t* own, const uint64_t* enemy, float* policy, float* value, size_t n,
                      cudaStream_t stream, float* dbg_tower, const uint32_t* n_dev = nullptr, float* dbg_logits = nullptr,
                      float* dbg_vlogit = nullptr);
// RZ_NET_IMPL_AUTO -> the implementation used for a batch of capacity n
int select_impl(const rz_net* net, size_t n, int impl);
int net_pack_tc(rz_net* net, cudaStream_t stream);
// the wgmma towers' launches on a network hold this lock: they share its residual scratch and head-feature buffer
std::mutex& tower_mutex();
// grows net->feat to at least n rows (under tower_mutex(); a reallocation synchronises the device first, since launches on
// other streams may still read the old buffer)
int head_features(rz_net* net, size_t n);
// the same tower for 64 and 128 filters, B = 512 / F boards per tile (rz_net_tc_narrow.cu)
int net_forward_tc_narrow(rz_net* net, const uint64_t* own, const uint64_t* enemy, float* policy, float* value, size_t n,
                          cudaStream_t stream, float* dbg_tower, const uint32_t* n_dev, float* dbg_logits, float* dbg_vlogit);
int net_pack_tc_narrow(rz_net* net, cudaStream_t stream);
inline bool tc_width(int filters) { return filters == 64 || filters == 128 || filters == 256; }
// thread-block clusters of the tower kernels: 2 = CTA pairs sharing the weight stages (default), 1 = single CTAs
int set_tower_cluster(int cluster);
int tower_cluster();   // the current setting: rz_net_set_tower_cluster, else RZ_TOWER_CLUSTER, else 2
int net_forward(rz_net* net, const uint64_t* own, const uint64_t* enemy, float* policy, float* value, size_t n, int impl,
                cudaStream_t stream);

}  // namespace rz
