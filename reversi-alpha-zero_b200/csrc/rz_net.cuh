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
    __half* tc_w;        // [2R layers][9 taps][F/8 kc][F n][8] fp16: input channel ci = 8 kc + j; a weight stage is a run of
                         // consecutive kc: F = 256: 8 kc (64 input channels of one tap, 32 KB); 128: one tap; 64: three taps
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

// optional outputs of the tensor-core towers, each nullable: fp32 tower output [n][64 pixels][F], policy logits [n][64]
// (before the softmax), value logit [n] (before the tanh)
struct TowerDebug {
    float* tower;
    float* logits;
    float* vlogit;
};
// policy [n][64] and value [n] of n positions (*n_dev of them when n_dev is set: a count known only on the device, <= n)
// by implementation impl (RZ_NET_IMPL_*; AUTO picks by n), on stream; debug needs a tensor-core tower
int net_forward(rz_net* net, const uint64_t* own, const uint64_t* enemy, float* policy, float* value, size_t n,
                const uint32_t* n_dev, int impl, cudaStream_t stream, const TowerDebug* debug);
// thread-block clusters of the throughput towers: 2 = CTA pairs sharing the weight stages (default), 1 = single CTAs
int set_tower_cluster(int cluster);
int tower_cluster();   // the current setting: rz_net_set_tower_cluster, else RZ_TOWER_CLUSTER, else 2

}  // namespace rz
