/*
 * rz_engine.h -- C ABI of librz_engine.so: the H100-native self-play hot path of reversi-alpha-zero.
 *
 * The reference (mokemokechicken/reversi-alpha-zero) has no FFI seam: its self-play path is Python
 * calling Python (SURVEY.md section 8(b)).  Each entry point below therefore names the reference
 * *Python* interface it replaces (path:line under /root/reference/src/reversi_zero/); the ctypes
 * binding a maintainer would add on the reference side is shown in INTEGRATION.md and is what
 * reversi-alpha-zero_b200/reversi_zero_b200/_cabi.py contains.
 *
 * Conventions
 *   - every function returns int: 0 (RZ_OK) or a negative RZ_E* code; rz_last_error() gives the
 *     thread-local message.  CUDA errors are captured and reported, never abort()ed.
 *   - plain pointers and sizes only; the caller owns every buffer it passes in.  `*_dev` functions
 *     take DEVICE pointers and a cudaStream_t (as void*, 0 = default stream) and are asynchronous;
 *     functions without the suffix take HOST pointers, stage through the library's own device
 *     buffers and return after the result is in the host buffer.
 *   - board encoding (lib/bitboard.py:11-17): uint64 bitboard, bit i = square y*8+x, bit 0 top-left.
 *   - Player: 1 = black, 2 = white (env/reversi_env.py:9); Winner: 0 = none, 1 = black, 2 = white,
 *     3 = draw (env/reversi_env.py:11).
 *   - handles are not thread-safe; one engine per GPU driven by one host thread (exception: rz_engine_poll, see there).
 */
#ifndef RZ_ENGINE_H
#define RZ_ENGINE_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define RZ_OK 0
#define RZ_EINVAL (-1)   /* bad argument */
#define RZ_ECUDA (-2)    /* CUDA runtime / launch error (message has the CUDA string) */
#define RZ_ENOMEM (-3)   /* host or device allocation failed */
#define RZ_ESTATE (-4)   /* call not valid in this state (e.g. weights not loaded) */
#define RZ_ECAPACITY (-5) /* an engine arena overflowed (nodes / edges / records) */
#define RZ_EIO (-6)      /* file I/O failed */

#define RZ_ABI_VERSION 2

int rz_abi_version(void);
const char* rz_last_error(void);
/* number of CUDA devices visible; RZ_ECUDA if the runtime cannot initialise. */
int rz_device_count(int* count);

/* ------------------------------------------------------------------------------------------------
 * K1 -- stateless batched bitboard operators (lib/bitboard.py, env/reversi_env.py).
 * ---------------------------------------------------------------------------------------------- */

/* legal-move mask per position.  Replaces lib/bitboard.py:53-67 find_correct_moves (+ :95-116). */
int rz_find_correct_moves_dev(const uint64_t* own, const uint64_t* enemy, uint64_t* out, size_t n, void* stream);
int rz_find_correct_moves(const uint64_t* own, const uint64_t* enemy, uint64_t* out, size_t n);

/* flipped-disc mask for a move at pos[i] (0..63); like the reference it does NOT check that pos is
 * empty or legal (returns 0 when nothing is outflanked).  Replaces lib/bitboard.py:70-92 calc_flip. */
int rz_calc_flip_dev(const uint8_t* pos, const uint64_t* own, const uint64_t* enemy, uint64_t* out, size_t n, void* stream);
int rz_calc_flip(const uint8_t* pos, const uint64_t* own, const uint64_t* enemy, uint64_t* out, size_t n);

/* one ReversiEnv.step per environment, structure-of-arrays, in place.  action[i] in 0..63, or -1 for
 * None (= resign).  Semantics of env/reversi_env.py:42-85: illegal move => mover loses; opponent
 * without a move => auto-pass; neither side can move => game over, winner by disc count.
 * legal_out (nullable) receives the legal-move mask of the side to move after the step (0 if done). */
int rz_step_dev(uint64_t* black, uint64_t* white, uint8_t* next_player, uint8_t* turn, uint8_t* done,
                uint8_t* winner, const int8_t* action, uint64_t* legal_out, size_t n, void* stream);
int rz_step(uint64_t* black, uint64_t* white, uint8_t* next_player, uint8_t* turn, uint8_t* done,
            uint8_t* winner, const int8_t* action, uint64_t* legal_out, size_t n);

/* board dihedral transform t in 0..7: flip_vertical if (t & 4), then (t & 3) x rotate90 -- the order
 * of agent/player.py:166-179 and :300-305.  Replaces lib/bitboard.py:119-159. */
int rz_dihedral_dev(const uint64_t* x, const uint8_t* t, uint64_t* out, size_t n, void* stream);

/* endgame solver (lib/alt/reversi_solver_cython.pyx:40-127 ReversiSolver.solve, the variant agent/player.py:15
 * imports), batched: for each position of the side to move, move[i] = best square and score[i] = its value in the
 * mover's frame.  exactly[i] != 0: exact final disc difference, first best move in ascending order; exactly[i] == 0:
 * win/loss/draw mode with the reference's early stop (only the sign of the score and the move are meaningful).
 * move[i] = -1 (score 0): no legal move, or more than 12 empty squares (the analogue of the reference's timeout,
 * after which ReversiPlayer falls back to the search). */
int rz_solve_dev(const uint64_t* own, const uint64_t* enemy, const uint8_t* exactly, int8_t* move, int8_t* score, size_t n,
                 void* stream);
int rz_solve(const uint64_t* own, const uint64_t* enemy, const uint8_t* exactly, int8_t* move, int8_t* score, size_t n);

/* Deep exact endgame solver (csrc/rz_solver_deep.cu): the exact mode of rz_solve for positions with up to 30 empty
 * squares, each solved by the whole current device (null-window probes over a split AND/OR tree, one lane per leaf).
 * Host arrays; the n positions are solved one after another; synchronous.  For each position in the mover's frame:
 * score[i] = exact final disc difference (empties not awarded), move[i] = first square in ascending order reaching it.
 * move[i] = -1 and score[i] = 0 when the mover has no legal move (a finished game included), the position has more
 * than 30 empties, or `timeout_s` seconds passed before the answer was proven (checked between slices, so a call
 * returns within the timeout plus one slice plus the host's split time).  stats: nullable, n entries.
 * Workspace: allocated on first use per device and kept (about 1.3 GB on a 132-SM H100: 240 MB of node table and parked
 * stacks, and the 1 GiB transposition table); one call per device at a time.  The transposition table holds proven
 * bounds only, shared by the probes of a call and kept across calls, so consecutive positions of one game reuse each
 * other's proofs; it changes the work, never an answer. */
typedef struct rz_deep_solve_stats {
    int32_t probes;      /* null-window probes (value and move) */
    int32_t slices;      /* kernel slices */
    int32_t resplits;    /* open leaves the host split again between slices */
    int32_t pad;
    int64_t leaves;      /* leaves of the split trees, summed over probes */
    int64_t node_steps;  /* node steps of the leaf machines */
    double seconds;      /* wall time of the position */
} rz_deep_solve_stats;
int rz_solve_deep(const uint64_t* own, const uint64_t* enemy, int8_t* move, int8_t* score, size_t n, double timeout_s,
                  rz_deep_solve_stats* stats);
/* rz_solve_deep with a stop flag owned by the caller (nullable; NULL is rz_solve_deep).  The flag is read before each
 * position and wherever the timeout is checked, and may be set from another thread: once it is nonzero the call returns
 * within one slice plus the host's split time, and every position not yet finished answers move -1, score 0, like a
 * timeout.  The transposition table only ever holds proven bounds, so a stopped solve leaves nothing a later solve of
 * the same position could be misled by. */
int rz_solve_deep_with_stop(const uint64_t* own, const uint64_t* enemy, int8_t* move, int8_t* score, size_t n, double timeout_s,
                            const volatile int32_t* stop, rz_deep_solve_stats* stats);
/* The value of every legal move of one position (own to move), for endgame hints: bounds lo[sq] <= value <= hi[sq] of
 * the move at sq, in the mover's frame (exact final disc difference, empties not awarded).  *legal receives the mover's
 * legal mask, and lo / hi are meaningful on its squares only (0 elsewhere); with no legal move or more than 30 empties
 * *legal = 0 and nothing is solved.  Every round is one forest with a root per open move at that move's own threshold
 * (1, then 0, then the middle of its bounds), at most 8 rounds.  n_best >= 0 (0: every move): a move stops being refined
 * once its hi is below the n_best-th largest lo.  On a normal return every move whose value is at least the n_best-th
 * best value (ties included) has lo == hi, and every other move has hi below that value.  A timeout or the stop flag
 * (nullable, as in rz_solve_deep_with_stop) ends the call within one slice plus the host's split time, with the bounds
 * proven so far, which always hold.  on_round (nullable) is called on the calling thread after every round with the
 * current bounds; it must not call back into the solver.  stats (nullable): `probes` counts the forests.  The rounds
 * probe and fill the transposition table like rz_solve_deep's probes. */
typedef void (*rz_deep_moves_cb)(const int8_t* lo, const int8_t* hi, void* user);
int rz_solve_deep_moves(uint64_t own, uint64_t enemy, int n_best, double timeout_s, const volatile int32_t* stop,
                        int8_t lo[64], int8_t hi[64], uint64_t* legal, rz_deep_moves_cb on_round, void* user,
                        rz_deep_solve_stats* stats);
/* Tuning of rz_solve_deep for tests and measurements: slice length (us), leaf target of the split and leaf floor
 * (empties below which the split stops); 0 restores each default (4000 us, one leaf per lane, 10 empties).  The next
 * call starts from an empty transposition table, so that it searches under the new tuning. */
int rz_solve_deep_tune(int slice_us, int leaf_target, int leaf_floor);
/* The deep solver's transposition table on the current device, for tests and measurements.  rz_solve_deep_table sets its
 * size (rounded down to a power of two of 128-byte buckets, at least one; 0 restores the default 1 GiB) from the next
 * rz_solve_deep call on, which then starts from an empty table, as after rz_solve_deep_tune.  rz_solve_deep_clear
 * empties the table and zeroes its counts now.  rz_solve_deep_table_stats: counts since the table was last emptied
 * (all zero before the first call). */
typedef struct rz_deep_table_stats {
    int64_t lookups;   /* frames looked up before they were searched */
    int64_t cutoffs;   /* ... decided by a stored bound, without search */
    int64_t hints;     /* ... that tried the stored best move first */
    int64_t stores;    /* decided frames written to a new entry */
    int64_t replaced;  /* ... of those, over another position's entry */
    int64_t merges;    /* decided frames merged into their position's entry */
    int64_t dropped;   /* stores dropped because another writer held the entry */
    int64_t occupied;  /* entries holding a position now */
    int64_t bytes;     /* table size */
} rz_deep_table_stats;
int rz_solve_deep_table(int64_t bytes);
int rz_solve_deep_clear(void);
int rz_solve_deep_table_stats(rz_deep_table_stats* out);

/* Every distinct opening of `plies` plies (1..12), enumerated on the current device (csrc/rz_openings.cu).  Two move
 * sequences are the same opening when they reach the same position up to the 8 board symmetries (transpositions
 * included); a sequence through a position whose side to move must pass, or whose game is over, is not an opening.  Each
 * opening is represented by the sequence that is least by (parent opening, move square) at every ply, in the orientation
 * that sequence reaches.  Output, host buffers, in ascending order of the canonical key (the least (own, enemy) pair over
 * the 8 images, own compared first): own[i] / enemy[i] = the position reached, in the mover's frame; moves[i * plies + j]
 * = its j-th move (square 0..63).  cap = 0: only *n_out is set (the outputs may be NULL); cap < *n_out: RZ_ECAPACITY.
 * level_counts (nullable, plies + 1 entries): the number of openings of 0 .. plies plies.  Repeated calls give identical
 * output.  Device memory grows with the level; a level that does not fit returns RZ_ENOMEM.  Synchronous. */
int rz_openings_enumerate(int plies, uint64_t* own, uint64_t* enemy, uint8_t* moves, size_t cap, size_t* n_out,
                          uint64_t* level_counts);
/* The opening book's graph (csrc/rz_openings.cu): every opening of 0 .. plies (1..10) plies and the moves between
 * consecutive levels, in CSR form.  Nodes, host buffers: level by level, each level exactly rz_openings_enumerate's
 * output for that many plies (ascending canonical key; level 0 is the initial position); own[i] / enemy[i] = the node in
 * its representative's orientation, mover's frame; key_hi[i] / key_lo[i] (nullable) = its canonical key.  level_counts
 * (nullable, plies + 1 entries) gives the level sizes.
 * Edges: node i's are edge_offset[i] .. edge_offset[i + 1] - 1 (edge_offset has *n_nodes + 1 entries; nodes of the last
 * level have none), one per legal move in ascending square order in the node's frame: edge_square = the square,
 * edge_child = the index within the next level of the child's class, or -1 when the child is not an opening (its mover
 * must pass, or the game is over).  cap_nodes = 0: only *n_nodes and *n_edges are set (the outputs may be NULL);
 * cap_nodes < *n_nodes or cap_edges < *n_edges: RZ_ECAPACITY.  Repeated calls give identical output; a level that does
 * not fit in device memory returns RZ_ENOMEM.  Synchronous. */
int rz_openings_book_graph(int plies, uint64_t* own, uint64_t* enemy, uint64_t* key_hi, uint64_t* key_lo, size_t cap_nodes,
                           size_t* n_nodes, uint64_t* level_counts, uint64_t* edge_offset, uint8_t* edge_square,
                           int32_t* edge_child, size_t cap_edges, size_t* n_edges);
/* The children of any n book nodes (csrc/rz_openings.cu): how an opening book grows beyond its full width and links a
 * level that rz_openings_book_graph did not build.  Inputs, host buffers: own[i] / enemy[i] = node i in the mover's frame;
 * next_hi / next_lo (NULL when n_next = 0) = the n_next ascending canonical keys of a sorted level.  Output, host buffers:
 * node i's children are edge_offset[i] .. edge_offset[i + 1] - 1 (edge_offset has n + 1 entries), one per legal move in
 * ascending square order: edge_square = the square; child_own / child_enemy = the child in the new mover's frame;
 * child_hi / child_lo = its canonical key; child_kind = 0 kept (an opening), 1 its mover must pass, 2 the game is over;
 * edge_child = the index of its key among next_hi / next_lo, or -1 when the child is not kept or not in that level.
 * edge_offset = NULL: only *n_edges is set (the other outputs may be NULL too); cap_edges < *n_edges: RZ_ECAPACITY.
 * Repeated calls give identical output.  Synchronous. */
int rz_openings_book_children(const uint64_t* own, const uint64_t* enemy, size_t n, const uint64_t* next_hi,
                              const uint64_t* next_lo, size_t n_next, uint64_t* edge_offset, uint8_t* edge_square,
                              int32_t* edge_child, uint64_t* child_own, uint64_t* child_enemy, uint64_t* child_hi,
                              uint64_t* child_lo, uint8_t* child_kind, size_t cap_edges, size_t* n_edges);

/* Scalar host twins for the single-environment Python objects (ReversiEnv / Board used by the
 * reference's evaluate.py, nboard.py, game_model.py): same header-only code as the device kernels
 * (csrc/rz_bitboard.cuh), compiled for the host.  Not a fallback for the batched path. */
typedef struct rz_env_state {
    uint64_t black, white;
    uint8_t next_player, turn, done, winner;
} rz_env_state;
uint64_t rz_find_correct_moves_host(uint64_t own, uint64_t enemy);
uint64_t rz_calc_flip_host(int pos, uint64_t own, uint64_t enemy);
uint64_t rz_dihedral_host(uint64_t x, int t);
/* Host twin of the BIT-SLICED formulation the batched GPU operators use (csrc/rz_bitsliced.cuh: 32 positions per thread,
 * one register per square): pos == NULL: out[i] = find_correct_moves(own[i], enemy[i]); else out[i] = calc_flip(pos[i], ..).
 * Same header compiled for the host; exists so that the formulation can be held against the oracle without a GPU. */
int rz_bitsliced_host(const uint8_t* pos, const uint64_t* own, const uint64_t* enemy, uint64_t* out, size_t n);
void rz_env_reset_host(rz_env_state* s);                                              /* reversi_env.py:26-32 */
void rz_env_update_host(rz_env_state* s, uint64_t black, uint64_t white, int next_player); /* :34-40 */
void rz_env_step_host(rz_env_state* s, int action /* -1 = None */);                   /* :42-74 */

/* ------------------------------------------------------------------------------------------------
 * NN -- policy/value residual CNN inference (agent/model.py:28-72 forward, agent/api.py:30-45).
 * ---------------------------------------------------------------------------------------------- */
typedef struct rz_net rz_net;

typedef struct rz_net_cfg {
    int32_t filters;     /* ModelConfig.cnn_filter_num   (config.py:189) */
    int32_t res_blocks;  /* ModelConfig.res_layer_num    (config.py:191) */
    int32_t value_fc;    /* ModelConfig.value_fc_size    (config.py:193) */
    int32_t kernel_size; /* ModelConfig.cnn_filter_size  (config.py:190); only 3 is supported */
} rz_net_cfg;

#define RZ_NET_IMPL_AUTO 0    /* wgmma tower when filters is 64, 128 or 256 and value_fc <= 512, else the generic kernel */
#define RZ_NET_IMPL_GENERIC 1 /* CUDA-core fp32 kernel, any configuration (the exact path) */
#define RZ_NET_IMPL_TCGEN05 2 /* fused persistent tensor-core (wgmma) tower, fp16 operands / fp32 accumulation (filters must
                                 be 64, 128 or 256, value_fc <= 512) */
#define RZ_NET_IMPL_SPLIT 3   /* the same tower with each 2-board tile split over an 8-CTA cluster: lower latency for small
                                 batches, bit-identical outputs (filters must be 256); AUTO picks it up to a measured batch size */

/* Thread-block clusters of the tensor-core tower from now on (process-wide): 2 = CTA pairs that share every weight stage
 * through cluster multicast (default; falls back to 1 where the GPU cannot hold a pair), 1 = single CTAs.  The default
 * comes from the environment variable RZ_TOWER_CLUSTER when the first network call is made. */
int rz_net_set_tower_cluster(int cluster);
int rz_net_create(const rz_net_cfg* cfg, int device, rz_net** out);
int rz_net_destroy(rz_net* net);
/* number of float32 values in the weight blob for this configuration.  Blob layout (Keras tensor
 * layouts, in this order): for conv0, then res{i}.conv1, res{i}.conv2 (i = 0..res_blocks-1):
 *   kernel[kh][kw][Cin][Cout], bias[Cout], bn_gamma, bn_beta, bn_mean, bn_var [Cout];
 * policy_conv (1x1, Cout = 2) same six tensors; policy_fc kernel[128][64], bias[64];
 * value_conv (1x1, Cout = 1) same six; value_fc1 kernel[64][V], bias[V]; value_fc2 kernel[V][1], bias[1].
 * BatchNormalization epsilon = 1e-3 (Keras default), inference statistics. */
int rz_net_blob_size(const rz_net* net, size_t* n_floats);
int rz_net_load_weights(rz_net* net, const float* blob_host, size_t n_floats);
/* same, blob already in device memory (e.g. after an NCCL broadcast from rank 0). */
int rz_net_load_weights_dev(rz_net* net, const float* blob_dev, size_t n_floats, void* stream);

/* batched forward from bitboards: plane 0 = own (side to move), plane 1 = enemy.
 * policy[n][64] softmax probabilities, value[n] tanh.  Device pointers. */
int rz_net_predict_dev(rz_net* net, const uint64_t* own, const uint64_t* enemy, float* policy, float* value,
                       size_t n, int impl, void* stream);
/* rz_net_predict_dev for a batch whose size is known only on the device: *count_dev (<= max_n) positions are evaluated,
 * and rows from *count_dev to max_n of policy and value are left as they were (the engine's leaf-batch path). */
int rz_net_predict_counted_dev(rz_net* net, const uint64_t* own, const uint64_t* enemy, float* policy, float* value,
                               const uint32_t* count_dev, size_t max_n, int impl, void* stream);
/* diagnostic variant of the tensor-core tower path: additionally writes the fp32 residual-tower output
 * tower[n][64 pixels][filters channels] (pixel = y*8+x) so tests can localise a numerical difference. */
int rz_net_debug_tower_dev(rz_net* net, const uint64_t* own, const uint64_t* enemy, float* policy, float* value,
                           float* tower, size_t n, void* stream);
/* same, plus the head outputs BEFORE softmax / tanh -- policy_logits[n][64] (the input of the policy_out softmax,
 * agent/model.py:47) and value_logit[n] (the input of the value_out tanh, :55) -- so that the north-star tolerance
 * ("policy/value logits within 1e-3") can be asserted on the logits themselves; tower may be NULL. */
int rz_net_debug_heads_dev(rz_net* net, const uint64_t* own, const uint64_t* enemy, float* policy, float* value,
                           float* tower, float* policy_logits, float* value_logit, size_t n, void* stream);
/* same, with the tower implementation chosen: RZ_NET_IMPL_AUTO, _TCGEN05 or _SPLIT. */
int rz_net_debug_heads_impl_dev(rz_net* net, const uint64_t* own, const uint64_t* enemy, float* policy, float* value,
                                float* tower, float* policy_logits, float* value_logit, size_t n, int impl, void* stream);
/* the implementation RZ_NET_IMPL_AUTO runs for a batch of n positions (on the engine's counted path: its capacity). */
int rz_net_select_impl(const rz_net* net, size_t n, int* impl);
/* ReversiModelAPI.predict (agent/api.py:30-45): planes uint8 [n][2][8][8] with values {0,1}, host
 * buffers in, policy[n][64] / value[n] host buffers out. */
int rz_net_predict(rz_net* net, const uint8_t* planes, float* policy, float* value, size_t n, int impl);

/* ------------------------------------------------------------------------------------------------
 * Engine -- on-device MCTS self-play (agent/player.py ReversiPlayer, worker/self_play.py).
 * ---------------------------------------------------------------------------------------------- */
typedef struct rz_engine rz_engine;

#define RZ_EVAL_NET 0  /* leaves evaluated by the rz_net */
#define RZ_EVAL_FAKE 1 /* deterministic test evaluator: policy 1/64, value (#own - #enemy)/64 */

typedef struct rz_engine_cfg {
    int32_t games;                  /* concurrent game slots on this GPU */
    int32_t simulation_num_per_move; /* PlayConfig.simulation_num_per_move (config.py:129) */
    int32_t parallel_search_num;    /* :141, <= 16 */
    int32_t virtual_loss;           /* :139 */
    int32_t change_tau_turn;        /* :138 */
    int32_t thinking_loop;          /* :132 */
    int32_t required_visit_to_decide_action; /* :133 */
    int32_t start_rethinking_turn;  /* :134 */
    int32_t allowed_resign_turn;    /* :145 */
    int32_t use_resign_threshold;   /* 0 => resign_threshold is None (:144) */
    int32_t share_mtcs_info;        /* share_mtcs_info_in_self_play (:130) */
    int32_t eval_mode;              /* RZ_EVAL_* */
    int32_t net_impl;               /* RZ_NET_IMPL_* */
    int32_t max_plies;              /* per-game ply log capacity, 0 => 64 */
    int32_t warm_start;             /* 1: the FIRST game of every slot begins after a random number (0..57) of
                                       random legal plies, so a fresh engine is in steady state (game phases
                                       spread uniformly) instead of all slots marching in lock step; those
                                       pre-played plies are not searched and not recorded */
    int32_t overlap_groups;         /* 0 = auto (2 when games >= 256), 1, or 2: slot groups whose MCTS tick overlaps
                                       the other group's network launch on a second stream */
    int32_t max_sims_per_wave;      /* simulations one game may START in one wave (0 = 2 x parallel_search_num).  Bounds
                                       the work of a wave for games whose simulations end in terminal positions without
                                       needing the network (endgame), so no slot delays the whole batch. */
    int32_t use_solver_turn;        /* PlayConfig.use_solver_turn (config.py:154): from this turn on the move is the exact
                                       endgame solution (agent/player.py:100-103,150-161) and the ply is not training data;
                                       0 = off.  Positions the device solver refuses (> 12 empties) are searched instead. */
    int32_t use_solver_turn_in_simulation; /* :155, agent/player.py:237-251: WLD-solved nodes inside the search; 0 = off.
                                       Solves are resumable: each wave advances the unfinished ones for at most
                                       RZ_SOLVER_BUDGET_US microseconds (environment, read by rz_engine_create; default
                                       2000) and a game waits until its solves are done -- results do not depend on it. */
    int32_t reset_mtcs_info_per_game; /* PlayConfig.reset_mtcs_info_per_game (config.py:131; worker/self_play.py:111-134): a
                                       slot keeps its statistics for this many consecutive games (0 / 1: every game starts
                                       empty, ch5.yml; mini.yml uses 3).  Arenas grow by the same factor. */
    int32_t max_searches_per_game;  /* sizes the per-game node arena: nodes = this x simulation_num_per_move;
                                       0 = 60 x min(thinking_loop, 2).  Rethinking (thinking_loop > 1) is skipped
                                       when the arena could no longer hold one search per remaining ply. */
    int32_t arena_simulation_num;   /* the largest simulation count rz_engine_set_simulation_num will be asked for during this
                                       engine's life (the maximum over schedule_of_simulation_num_per_move and .force-sim,
                                       worker/self_play.py:262-272); the arenas are sized for it.  0 = simulation_num_per_move. */
    int32_t eval_cache_mb;          /* device memory (MiB) of the evaluation cache: a leaf whose transformed board the network
                                       evaluated before (in any game, with the weights now loaded) takes that result instead of
                                       a tower row -- the same bits, so the games do not change.  0 = the environment variable
                                       RZ_EVAL_CACHE_MB if set (read by rz_engine_create), else 2048; < 0 = off.  Always off
                                       with RZ_EVAL_FAKE and while a second network is set.  Loading new weights into the
                                       engine's network invalidates every entry. */
    float c_puct;                   /* :135 */
    float noise_eps;                /* :136 */
    float dirichlet_alpha;          /* :137 */
    float resign_threshold;         /* :144 */
    float disable_resignation_rate; /* :146 */
    uint64_t seed;                  /* Philox key */
    uint64_t first_game_id;         /* ids handed to slots: first_game_id + k * game_id_stride */
    uint64_t game_id_stride;        /* (rank-strided sharding across GPUs, SURVEY 8(e)) */
    uint64_t max_games;             /* stop starting new games after this many (0 = unlimited) */
} rz_engine_cfg;

/* one decided ply of a finished game (compact form of what ReversiPlayer.moves holds,
 * agent/player.py:166-179; the 8 symmetries are expanded by rz_write_play_data). */
typedef struct rz_ply {
    uint64_t own, enemy;  /* position in the mover's frame */
    int32_t n_visit[64];  /* root visit counts N(s,a) at decision time */
    int16_t action;       /* 0..63, -1 = resigned */
    uint8_t player;       /* 1 black / 2 white */
    uint8_t loops;        /* thinking loops used */
    uint8_t recorded;     /* 1 if this ply is training data (0 for a resignation) */
    uint8_t pad;
    uint16_t waves;       /* engine waves this slot spent deciding the ply (saturating; measurement only, no reference twin) */
    float n;              /* ActionWithEvaluation.n */
    float q;              /* ActionWithEvaluation.q */
} rz_ply;

typedef struct rz_game {
    uint64_t game_id;
    uint64_t black, white;  /* final position */
    int32_t first_ply;      /* index into the ply array returned by the same poll */
    int32_t n_plies;
    int32_t expansions;     /* NN evaluations spent on this game */
    int32_t simulations;
    uint8_t winner;         /* Winner enum */
    int8_t black_z;         /* +1 / -1 / 0 */
    uint8_t resign_enabled;
    uint8_t resigned_mask;  /* bit0 black wanted to resign, bit1 white */
    uint8_t turn;           /* ReversiEnv.turn at the end */
    uint8_t black_net;      /* matches and leagues: index of the network that played black (0 in self-play) */
    uint8_t white_net;      /* ... and white (0 in self-play, 1 - black_net in a two-network match) */
    uint8_t opening_plies;  /* plies of the opening the game started from (rz_engine_set_openings; 0 without one) */
    int32_t table_nodes;    /* positions in the slot's statistics table at the end of the game (half of the reference's
                               len(mtcs_info.var_p), which also holds every colour-swapped mirror key, worker/self_play.py:127) */
    int32_t pad2;
} rz_game;

typedef struct rz_stats {
    uint64_t games_started, games_finished;
    uint64_t expansions;    /* leaves evaluated == "node expansions" */
    uint64_t simulations;
    uint64_t waves;
    uint64_t plies;
    uint64_t nn_launches, mcts_launches; /* kernels launched by the engine */
    uint64_t max_nodes_used, max_edges_used;
    double nn_ms, mcts_ms; /* device time (CUDA events on the engine's stream) spent in the two kernel families */
    double run_ms;         /* device time from the first to the last wave of each rz_engine_run call, accumulated */
    uint64_t tower_rows;    /* leaves the evaluator ran (expansions counts every evaluated leaf, cache hits included) */
    uint64_t cache_lookups; /* leaves looked up in the evaluation cache */
    uint64_t cache_hits;    /* ... served from it (hit counts of a two-group engine depend on timing; results do not) */
    uint64_t cache_repeats; /* tower rows not stored because their board was already in the cache when the wave's rows were
                               inserted: boards that two leaves of the same wave sent to the tower */
} rz_stats;

int rz_engine_create(const rz_engine_cfg* cfg, rz_net* net /* may be NULL for RZ_EVAL_FAKE */, int device,
                     rz_engine** out);
int rz_engine_destroy(rz_engine* e);
/* run waves until at least `finished_target` games (cumulative) have finished or `max_waves` waves
 * were executed (0 = no limit).  Finished games accumulate in a host-side queue until polled.
 * rz_engine_poll (and only it) may be called from a second host thread while rz_engine_run is in progress: the queue is
 * a mutex-protected single-producer / single-consumer hand-off, which is how the worker's writer thread overlaps
 * harvesting and play_data output with the waves (the reference overlaps through processes, worker/self_play.py:36-41). */
int rz_engine_run(rz_engine* e, uint64_t finished_target, uint64_t max_waves);
/* pop up to game_cap finished games (and their plies, up to ply_cap) from the queue. */
int rz_engine_poll(rz_engine* e, rz_game* games, size_t game_cap, size_t* n_games, rz_ply* plies, size_t ply_cap,
                   size_t* n_plies);
int rz_engine_stats(rz_engine* e, rz_stats* out);
/* the cache_lookups / cache_hits of rz_stats split by the turn of the searched root: n must be 61; entry t < 60 counts
 * searches at turn t, entry 60 every search of the first game of a slot of a warm_start engine (random pre-played
 * openings, which rarely repeat). */
int rz_engine_cache_turn_stats(rz_engine* e, uint64_t* lookups, uint64_t* hits, int n);
/* no slot starts a game whose local index (slot + games already started by the slot x games) is >= max_games; 0 = no
 * limit, 1 = let the resident games finish and start nothing (rz_engine_run then returns when every slot is idle). */
int rz_engine_set_max_games(rz_engine* e, uint64_t max_games);
/* warm_start only: weight[t] (t = 0 .. n-1, n <= 60) is proportional to the time a game spends at turn t; the first
 * game of every slot then begins at turn t with probability weight[t] / sum and its first search runs a uniformly drawn
 * fraction of simulation_num_per_move (of the waves the profile gives the turn, where that is less), i.e. the slots start in the stationary state of an engine that has been running
 * for a long time (used by bench.py, which measures finished games per second over a window shorter than a game).
 * Without this call the turns 0..57 are equally likely.  Call before the first rz_engine_run. */
int rz_engine_set_warm_start_profile(rz_engine* e, const float* weight, int n);
/* change the per-move simulation count for games started from now on
 * (SelfPlayWorker.decide_simulation_num_per_move, worker/self_play.py:262-272). */
int rz_engine_set_simulation_num(rz_engine* e, int32_t sims);
/* evaluation matches (worker/evaluate.py:44-96: best model vs challenger): with a second network set, the game with
 * local index i is played by the first network as black when i is even and by the second when i is odd (the
 * reference draws the colours at random, :70), and every search is evaluated by the mover's own network.  Use
 * share_mtcs_info = 0 (the reference gives each evaluation player its own statistics).  RZ_EVAL_FAKE: the "second
 * network" is the deterministic evaluator with the value negated.  NULL switches back to one network.  Call before
 * the first rz_engine_run. */
int rz_engine_set_second_net(rz_engine* e, rz_net* net_b, int enable);
/* leagues: up to RZ_MAX_NETS networks in one engine.  The game with local index i (< n_games) is played by
 * nets[black_net[i]] as black and nets[white_net[i]] as white; every search is evaluated by the mover's own network, each
 * network by its own implementation (widths and depths may differ).  The table (2 bytes per game) is copied to the
 * device.  RZ_EVAL_FAKE: nets may be NULL, and network k is the deterministic evaluator with its value multiplied by
 * fake_scale[k] (NULL: all 1).  rz_engine_set_second_net is the two-network case with no table (colours alternate with
 * the local index, scales 1 and -1).  The evaluation cache stays off while more than one network is set.  Row buffers
 * grow to n_nets x games x parallel_search_num rows (RZ_ENOMEM if that fails).  RZ_EINVAL, with the engine unchanged:
 * n_nets outside 2..RZ_MAX_NETS, an index >= n_nets, a NULL network under RZ_EVAL_NET, max_games 0 or greater than
 * n_games (rz_engine_set_max_games then keeps to that bound), or a call after the first wave. */
#define RZ_MAX_NETS 16
int rz_engine_set_nets(rz_engine* e, rz_net* const* nets, const float* fake_scale, int n_nets, const uint8_t* black_net,
                       const uint8_t* white_net, uint64_t n_games);
/* update the resignation rule for decisions taken from now on (SelfPlayWorker's threshold auto-tuner,
 * worker/self_play.py:250-260). */
/* games from openings: the game with local index i (< n_games) starts after the n_moves[i] squares at
 * moves[i * RZ_MAX_OPENING_PLIES ...], which the engine plays without a search and does not record; n_moves[i] = 0 is the
 * initial position (a table of zeros gives the games of no table).  The game's turn and side to move then follow from the
 * opening (change_tau_turn, allowed_resign_turn and use_solver_turn count from the initial position), a game with an
 * opening has no forced first move, its statistics start empty at the opening's position, and rz_game.opening_plies
 * reports the length.  Works with one network, rz_engine_set_second_net and rz_engine_set_nets.  RZ_EINVAL, with the engine
 * unchanged: an illegal move, a move after which the other side must pass, a move that ends the game, more than
 * RZ_MAX_OPENING_PLIES moves, max_games 0 or greater than n_games (rz_engine_set_max_games then keeps to that bound),
 * warm_start on, or a call after the first wave. */
#define RZ_MAX_OPENING_PLIES 20
int rz_engine_set_openings(rz_engine* e, const uint8_t* moves, const uint8_t* n_moves, uint64_t n_games);
int rz_engine_set_resign_threshold(rz_engine* e, int use_resign_threshold, float resign_threshold);
/* single-position search (ReversiPlayer.action outside the self-play loop: evaluate.py, nboard.py, GUI; also the
 * parity-test hook): every slot searches (own, enemy) with `player` to move for simulation_num_per_move
 * simulations; returns the root statistics of slot `slot`: n_visit[64], w_sum[64] (mover's frame).
 * keep_tree != 0 keeps the slot's transposition table from earlier calls (the reference's MCTSInfo that
 * persists across the moves of a game, agent/player.py:44-47); 0 starts from an empty table. */
int rz_engine_search_root(rz_engine* e, uint64_t own, uint64_t enemy, int player, int slot, int keep_tree,
                          int32_t* n_visit, float* w_sum);
/* one root per slot (whole-game analysis): slot i < n searches (own[i], enemy[i]) -- host arrays, mover's frame -- with
 * player[i] (1 or 2) to move for simulation_num_per_move simulations; slots n .. games-1 stay idle and take no tower rows.
 * keep_tree as in rz_engine_search_root, per slot, so repeated calls with keep_tree = 1 continue every slot's tree (a
 * search in chunks).  Returns the root statistics of the n slots: n_visit[n][64], w_sum[n][64].  With noise_eps = 0 every
 * slot uses the game id first_game_id, so slot i gives the same bits as a one-slot engine of the same configuration
 * running rz_engine_search_root on that position, whatever the other slots hold; with root noise, slot i uses the game
 * id first_game_id + i * game_id_stride (a one-slot engine created with that first_game_id reproduces it).
 * RZ_EINVAL, with the engine left usable: n outside 1..games, a player other than 1 or 2, or a root without a legal
 * move for its mover (passes and finished games are the caller's). */
int rz_engine_search_roots(rz_engine* e, const uint64_t* own, const uint64_t* enemy, const uint8_t* player, int n,
                           int keep_tree, int32_t* n_visit, float* w_sum);

/* ------------------------------------------------------------------------------------------------
 * play_data writer -- the reference's output contract (worker/self_play.py:180-194,
 * lib/data_helper.py:23-25): one JSON array of [[own, enemy], [p0..p63], z] records, all of black's
 * records of a game then all of white's, each recorded ply expanded to its 8 symmetries in the order
 * of agent/player.py:166-179.  Written to path + ".tmp" and renamed.  save_policy_of_tau_1 /
 * change_tau_turn select the stored policy exactly as agent/player.py:132,366-385.
 * ---------------------------------------------------------------------------------------------- */
int rz_write_play_data(const char* path, const rz_game* games, size_t n_games, const rz_ply* plies,
                       int save_policy_of_tau_1, int change_tau_turn, size_t* n_records);

/* ------------------------------------------------------------------------------------------------
 * Trainer-side ingest (SURVEY 8(f).4) -- replaces the pure-Python per-record loop of
 * OptimizeWorker.convert_to_training_data (worker/optimize.py:215-231) applied to
 * read_game_data_from_file (lib/data_helper.py:28-30).
 *
 * A "play row" is one recorded ply before the 8-symmetry expansion: 280 bytes instead of ~5 KB of JSON text.
 * rz_write_play_rows writes the rows of the same games, in the same order, as rz_write_play_data writes records
 * (file: 32-byte header {"RZROWS\0\1", int32 save_policy_of_tau_1, int32 change_tau_turn, uint64 n_rows, 8 bytes 0}
 * + n_rows rows).  rz_ingest[_dev] expands rows into the arrays the reference trainer builds from the JSON file:
 *   planes [8*n_rows][2][8][8] uint8   == np.array(state_list)   (bit_to_array, lib/bitboard.py:136-138)
 *   policy [8*n_rows][64]      float32 == np.array(policy_list) rounded to the float32 Keras feeds the model
 *   z      [8*n_rows]          float32 == np.array(z_list)
 * row r, symmetry t (t = flip*4 + rot, agent/player.py:166-179) -> output record 8*r + t.
 * ---------------------------------------------------------------------------------------------- */
typedef struct rz_play_row {
    uint64_t own, enemy;  /* position in the mover's frame */
    int32_t n_visit[64];  /* root visit counts at decision time */
    int32_t z;            /* game result from the mover's point of view: +1 / 0 / -1 */
    int32_t pad;
} rz_play_row;

int rz_write_play_rows(const char* path, const rz_game* games, size_t n_games, const rz_ply* plies,
                       int save_policy_of_tau_1, int change_tau_turn, size_t* n_rows);
/* rows == NULL: only report n_rows and the two policy settings stored in the header */
int rz_read_play_rows(const char* path, rz_play_row* rows, size_t capacity, size_t* n_rows,
                      int* save_policy_of_tau_1, int* change_tau_turn);
int rz_ingest_dev(const rz_play_row* rows, size_t n_rows, int save_policy_of_tau_1, int change_tau_turn,
                  uint8_t* planes, float* policy, float* z, void* stream);   /* device pointers */
int rz_ingest(const rz_play_row* rows, size_t n_rows, int save_policy_of_tau_1, int change_tau_turn,
              uint8_t* planes, float* policy, float* z);                       /* host pointers */

/* play_*.json text -> the same three arrays, one output record per JSON record, in file order:
 *   planes [n][2][8][8] uint8 = bit_to_array(own), bit_to_array(enemy); policy [n][64] and z [n] float32 =
 *   float32(float64(text)) -- Python's correctly rounded float(), then round-to-nearest-even to float32.
 * The text must be one JSON array of [[own, enemy], [p0, ..., p63], z] records: bitboards are integer literals in
 * [0, 2^64) (refused otherwise, never truncated), the other 65 values JSON numbers or NaN / Infinity / -Infinity, any
 * JSON whitespace between tokens.  Anything else -- a string, a wrong arity, a missing bracket, trailing bytes, a
 * truncated file -- returns RZ_EINVAL with *error_offset = the byte offset of the first error (else (size_t)-1).
 * *n_records is always set once the records are counted; if it exceeds `capacity` the call returns RZ_ECAPACITY and
 * writes nothing, so a call with capacity 0 and null outputs sizes the buffers.
 * rz_ingest_json_dev: text and outputs in device memory; runs on `stream` and synchronises it (the record count is
 * read back to size the parse; records the device cannot round exactly are converted on the host and patched).
 * rz_ingest_json_host: the host twin (same parser, host pointers).  rz_ingest_json: reads the file at `path`, host
 * outputs, through the device parser (it reads the file twice when sized with capacity 0 first). */
int rz_ingest_json_dev(const char* text, size_t n_bytes, size_t capacity, uint8_t* planes, float* policy, float* z,
                       size_t* n_records, size_t* error_offset, void* stream);
int rz_ingest_json_host(const char* text, size_t n_bytes, size_t capacity, uint8_t* planes, float* policy, float* z,
                        size_t* n_records, size_t* error_offset);
int rz_ingest_json(const char* path, size_t capacity, uint8_t* planes, float* policy, float* z, size_t* n_records,
                   size_t* error_offset);

/* ------------------------------------------------------------------------------------------------
 * Trainer -- one SGD step of the network on the device (worker/optimize.py:73-86 OptimizeWorker.train_epoch ->
 * Keras fit on agent/model.py:28-72,104-110).  Training-mode BatchNormalization (batch statistics, biased variance,
 * epsilon 1e-3); loss = batch mean of sum -y log(p + 1e-7) + batch mean of (v - z)^2 + l2_reg * sum of squared Conv2D /
 * Dense kernels; Keras SGD: v = momentum * v - lr * g, w = w + v for kernels, biases and BN gamma / beta; BN moving
 * statistics: moving = bn_momentum * moving + (1 - bn_momentum) * batch statistic.  3x3 convolutions use TF32 operands
 * with fp32 accumulation; every reduction has a fixed order, so equal inputs give bit-identical weights.
 * Configurations: filters a multiple of 16 in [16, 256], kernel_size 3, res_blocks in [0, 64], value_fc in [1, 4096]
 * (else RZ_EINVAL).
 * ---------------------------------------------------------------------------------------------- */
typedef struct rz_trainer rz_trainer;

typedef struct rz_train_cfg {
    int32_t max_batch;  /* largest batch rz_trainer_step_dev will be given (sizes the saved activations) */
    float momentum;     /* SGD(momentum=0.9), worker/optimize.py:84 */
    float l2_reg;       /* ModelConfig.l2_reg (config.py:192) */
    float bn_momentum;  /* Keras BatchNormalization momentum, 0.99 */
} rz_train_cfg;

int rz_trainer_create(const rz_net_cfg* net, const rz_train_cfg* cfg, int device, rz_trainer** out);
/* A data-parallel group of 1 <= n_devices <= 64 replicas on devices[0..n) (repeats allowed); devices[0] is the primary.
 * Every rz_trainer_* call below takes either kind of handle, and a group's step gives exactly the bits of a single
 * trainer's step on the same batch.  rz_trainer_step_dev splits the batch into contiguous shards, one per replica, whose
 * boundaries sit on the weight-gradient split grid of the F->F convolutions (conv0's without residual blocks), as even
 * as that grid allows (rz_train_shard_plan_host); a replica may get an empty shard.  Only the batch's own records leave
 * the primary.  The replicas exchange per-record BatchNorm partials, per-record head tensors and weight-gradient split
 * partials and add them in the single trainer's order; every replica then applies the same gradient, so weights,
 * momentum and moving statistics stay identical.  The dataset, index, loss and stream are the primary's; the other
 * replicas run on streams the trainer owns and join the caller's stream at the end of the step.  load_weights[_dev]
 * load every replica; weights_dev, last_grad_dev and debug_conv_dev use the primary.  cfg->max_batch bounds the global
 * batch.  n_devices == 1 is rz_trainer_create(devices[0]).  RZ_EINVAL for an ordinal outside the visible devices. */
int rz_trainer_create_group(const rz_net_cfg* net, const rz_train_cfg* cfg, const int* devices, int n_devices, rz_trainer** out);
/* the shards of a group step: replica r trains on batch positions [bounds[r], bounds[r + 1]); bounds has n_devices + 1 */
int rz_train_shard_plan_host(int filters, int res_blocks, int batch, int n_devices, int32_t* bounds);
int rz_trainer_destroy(rz_trainer* t);
/* same count as rz_net_blob_size for the same configuration */
int rz_trainer_blob_size(const rz_trainer* t, size_t* n_floats);
/* weights in the blob layout of rz_net_load_weights; both also zero the momentum */
int rz_trainer_load_weights(rz_trainer* t, const float* blob_host, size_t n_floats);
int rz_trainer_load_weights_dev(rz_trainer* t, const float* blob_dev, size_t n_floats, void* stream);
/* current weights, blob layout (ready for rz_net_load_weights_dev or a model_weight.rzblob.npy file) */
int rz_trainer_weights_dev(rz_trainer* t, float* blob_dev, size_t n_floats, void* stream);
/* one step on records index[0..batch) of the device arrays planes[n_records][2][8][8] u8, policy[n_records][64] f32,
 * z[n_records] f32 (what rz_ingest_dev writes); 1 <= batch <= max_batch; indices may repeat.  loss_dev[3] (device) =
 * total, policy, value loss of the batch before the update.  Asynchronous: no host synchronisation.  An index outside
 * [0, n_records) is never read: the step then leaves the weights unchanged and writes NaN losses. */
int rz_trainer_step_dev(rz_trainer* t, const uint8_t* planes, const float* policy, const float* z, size_t n_records,
                        const int32_t* index, size_t batch, float lr, float* loss_dev, void* stream);
/* test hook: gradient of the last step's total loss in blob layout (0 in the moving-statistics slots) */
int rz_trainer_last_grad_dev(rz_trainer* t, float* grad_dev, size_t n_floats, void* stream);
/* test hook: replica r's weights and momentum (blob layout) into blob_dev / vel_dev on the primary's device; r = 0 is the
 * primary, and a single trainer has only replica 0 */
int rz_trainer_replica_state_dev(rz_trainer* t, int r, float* blob_dev, float* vel_dev, size_t n_floats, void* stream);

/* test hook: one of the step's 3x3-convolution GEMMs on caller buffers (device pointers, pixel-major [M = 64 * batch][C]),
 * through the step's own kernels, weight images and weight-gradient split-K for this batch.  F = filters; kernels are in
 * blob layout [9 taps = kh*3+kw][Cin][Cout]; bias [F] and add [M][F] are optional (NULL) where not required.
 *   RZ_TRAIN_CONV0_FWD:   out[M][F] = conv(in[M][16], kernel[9][2][F]) + bias + add; in's channels 2..15 meet the zero
 *                         padding of the weight image
 *   RZ_TRAIN_CONV_FWD:    out[M][F] = conv(in[M][F], kernel[9][F][F]) + bias + add
 *   RZ_TRAIN_CONV_DGRAD:  out[M][F] = input gradient of that convolution for dy = in (through the mirrored, transposed
 *                         weight image) + bias + add; the step passes the skip connection's gradient as add
 *   RZ_TRAIN_CONV_WGRAD:  out[9][F][F] = weight gradient for input in[M][F] and dy = add[M][F] (kernel and bias NULL)
 *   RZ_TRAIN_CONV0_WGRAD: out[9][2][F] = the same for conv0's input in[M][16]
 * Uses the trainer's scratch (the step rewrites it), so it must be stream-ordered with the steps; allocates nothing.
 * RZ_EINVAL for batch outside [1, max_batch], a missing pointer or an unknown op. */
#define RZ_TRAIN_CONV0_FWD 0
#define RZ_TRAIN_CONV_FWD 1
#define RZ_TRAIN_CONV_DGRAD 2
#define RZ_TRAIN_CONV_WGRAD 3
#define RZ_TRAIN_CONV0_WGRAD 4
int rz_trainer_debug_conv_dev(rz_trainer* t, int op, const float* in, const float* kernel, const float* bias, const float* add,
                              size_t batch, float* out, void* stream);

/* test hook: copy one intermediate tensor of the last step (batch B, M = 64 * B pixel rows, L = 1 + 2 * res_blocks tower
 * layers) into out (device, exactly n_floats floats, stream-ordered after the step).  `layer` selects the tower layer
 * of Y, A, G, DY and DZ, the statistics slot of STATS, and is 0 for the others.  Single trainers only: RZ_ESTATE on a
 * group, before the first step, and for G / DY / DZ unless the last step ran with rz_trainer_debug_keep_backward on;
 * RZ_EINVAL for an unknown tensor, a layer out of range or a wrong n_floats. */
#define RZ_TRAIN_T_X0 0       /* [M][16] input planes, channels 2..15 zero */
#define RZ_TRAIN_T_Y 1        /* [M][F] conv output of tower layer l (pre-BN, bias included) */
#define RZ_TRAIN_T_A 2        /* [M][F] output of tower layer l (after BN, residual and ReLU) */
#define RZ_TRAIN_T_STATS 3    /* [4][F] slot l in [0, L + 2) (L: policy head, L + 1: value head): batch mean [F],
                                 invstd [F], then sum dz [C] and sum dz * xhat [C] packed after them, over the slot's
                                 C channels (F in the tower, 2 and 1 in the heads) */
#define RZ_TRAIN_T_STAT 4     /* [blob floats] the batch mean / biased variance the moving averages take, at the moving
                                 statistics' blob offsets; 0 elsewhere */
#define RZ_TRAIN_T_HC 5       /* [M][3] head 1x1 conv outputs (policy 0..1, value 2) */
#define RZ_TRAIN_T_AH 6       /* [M][3] their BN + ReLU outputs */
#define RZ_TRAIN_T_DH 7       /* [M][3] gradient of ah */
#define RZ_TRAIN_T_DYH 8      /* [M][3] gradient of hc */
#define RZ_TRAIN_T_HP 9       /* [B][128] policy Dense input (channels-first flatten of ah) */
#define RZ_TRAIN_T_HV 10      /* [B][64] value Dense input */
#define RZ_TRAIN_T_DL 11      /* [B][64] gradient of the logits */
#define RZ_TRAIN_T_H1 12      /* [B][V] value hidden layer (after ReLU) */
#define RZ_TRAIN_T_DH1 13     /* [B][V] its gradient below the ReLU */
#define RZ_TRAIN_T_DV 14      /* [B] gradient of the value output before tanh */
#define RZ_TRAIN_T_LP 15      /* [B] policy loss per record */
#define RZ_TRAIN_T_LV 16      /* [B] value loss per record */
#define RZ_TRAIN_T_LOSS_PV 17 /* [2] batch-mean policy and value loss */
#define RZ_TRAIN_T_G 18       /* [M][F] gradient of A(l)        (backward taps) */
#define RZ_TRAIN_T_DY 19      /* [M][F] gradient of Y(l)        (backward taps) */
#define RZ_TRAIN_T_DZ 20      /* [M][F] gradient below the ReLU that the skip connection carries, conv2 layers
                                 (l = 2, 4, ..) only        (backward taps) */
int rz_trainer_debug_tensor_dev(rz_trainer* t, int which, int layer, float* out, size_t n_floats, void* stream);
/* test hook: on != 0 allocates [L][3][64 * max_batch][F] floats and makes every following step copy each tower layer's
 * G, DY and DZ there (three device-to-device copies per layer); 0 frees them, and the step enqueues nothing extra.
 * RZ_ESTATE on a group. */
int rz_trainer_debug_keep_backward(rz_trainer* t, int on);

#ifdef __cplusplus
}
#endif
#endif /* RZ_ENGINE_H */
