// rz_engine_warp.cuh -- warp-per-game cooperative version of the MCTS tick (included by rz_engine.cu).
//
// Same state machine and the same arithmetic, operation for operation, as the thread-per-slot `Ctx`
// (which stays as a cross-check, RZ_TICK_IMPL=thread), but one WARP owns one game slot:
//   * control flow and all scalar state are warp-uniform (every lane computes the same values from the same
//     loads; lane 0 alone performs the stores / atomics, followed by __syncwarp() before anything re-reads them),
//     so the 32 lanes never diverge -- in the thread-per-slot kernel 32 different games share a warp and their
//     data-dependent loops serialise;
//   * the wide loops are spread over the lanes: PUCT over a node's children (one child per lane, warp arg-max
//     with first-index tie-break == the sequential strict '>' scan), Dirichlet noise (one Gamma draw per lane),
//     the 64-square policy gather + numpy-order re-normalisation (two squares per lane, column sums by ordered
//     shuffles), edge initialisation, backup (one path edge per lane) and the ply-log scatter.
// 4096 slots -> 4096 warps (131 k threads) instead of 128 warps: the kernel is latency-bound pointer chasing, so
// this is what lets the GPU overlap the dependent loads of different games.
#pragma once

struct WCtx {
    const DevCfg& c;
    const DevPtrs& p;
    const int s, lane;
    Slot sl;               // uniform working copy, written back by lane 0 at the end of the tick
    uint8_t dstat[kMaxK];  // uniform working copy of the descents' status
    Descent* desc;
    uint32_t* hash;
    Node* nodes;
    Edge* edges;
    static constexpr unsigned kFull = 0xffffffffu;

    __device__ WCtx(const DevCfg& c_, const DevPtrs& p_, int s_, int lane_)
        : c(c_), p(p_), s(s_), lane(lane_), sl(p_.slots[s_]), desc(p_.desc + (size_t)s_ * c_.K), hash(p_.hash + (size_t)s_ * c_.hash_cap),
          nodes(p_.nodes + (size_t)s_ * c_.nodes_cap), edges(p_.edges + (size_t)s_ * c_.edges_cap) {
        for (int k = 0; k < kMaxK; ++k) dstat[k] = k < c_.K ? desc[k].status : (uint8_t)D_PENDING;
    }
    __device__ void write_back() {
        if (lane == 0) {
            p.slots[s] = sl;
            for (int k = 0; k < c.K; ++k) desc[k].status = dstat[k];
        }
        __syncwarp();
    }

    __device__ void fail(int code) { if (lane == 0) atomicMin(&p.status->error, code); }
    __device__ uint32_t kpid_of(int pid) const { return c.share ? 0u : (uint32_t)pid; }

    __device__ int find_node(u64 own, u64 enemy, uint32_t kpid) const {
        const uint32_t mask = c.hash_cap - 1;
        uint32_t h = hash_key(own, enemy, kpid) & mask;
        for (uint32_t probe = 0; probe < c.hash_cap; ++probe) {
            const uint32_t e = hash[h];
            if ((e >> 20) != sl.gen) return -1;
            const uint32_t idx = (e & 0xFFFFFu) - 1;
            const Node& nd = nodes[idx];
            if (nd.own == own && nd.enemy == enemy && nd.kpid == kpid) return (int)idx;
            h = (h + 1) & mask;
        }
        return -1;
    }

    __device__ int create_node(u64 own, u64 enemy, uint32_t kpid) {
        const u64 legal = find_correct_moves(own, enemy);
        const uint32_t nl = (uint32_t)popc64(legal);
        if (sl.n_nodes >= c.nodes_cap || sl.n_edges + nl > c.edges_cap || sl.n_nodes >= 0xFFFFEu) { fail(RZ_ECAPACITY); return -1; }
        const uint32_t idx = sl.n_nodes++;
        if (lane == 0) {
            Node nd; nd.own = own; nd.enemy = enemy; nd.legal = legal; nd.edge_base = sl.n_edges; nd.exp = 0; nd.kpid = (uint8_t)kpid; nd.pad = 0;
            nodes[idx] = nd;
        }
        for (uint32_t i = lane; i < nl; i += 32) edges[sl.n_edges + i] = Edge{0, 0.f, 0.f, 0};
        sl.n_edges += nl;
        const uint32_t mask = c.hash_cap - 1;
        uint32_t h = hash_key(own, enemy, kpid) & mask;
        while ((hash[h] >> 20) == sl.gen) h = (h + 1) & mask;
        if (lane == 0) hash[h] = (sl.gen << 20) | (idx + 1);
        __syncwarp();
        return (int)idx;
    }

    // player.py:276-280; `path` lives in global memory (written by lane 0 during the descent)
    __device__ void backup(const uint32_t* path, int path_len, float v_root) {
        const float vl = (float)c.vl;
        for (int i = lane; i < path_len; i += 32) {
            Edge& e = edges[path[i] & 0x7FFFFFFFu];
            e.n += 1 - c.vl;
            const float sv = (path[i] >> 31) ? v_root : -v_root;
            e.w = e.w + (vl + sv);
        }
        __syncwarp();
    }

    __device__ double gamma_draw(uint32_t rootsel, uint32_t child) const {  // identical to Ctx::gamma_draw
        const double alpha = (double)c.alpha;
        const double a = alpha < 1.0 ? alpha + 1.0 : alpha;
        const double dd = a - 1.0 / 3.0, cc = 1.0 / sqrt(9.0 * dd);
        for (uint32_t att = 0; att < 16; ++att) {
            const U4 r = draw(c.seed, sl.game_id, rootsel, P_NOISE, child * 16 + att);
            const double z = sqrt(-2.0 * log(u01(r.x))) * cospi(2.0 * u01(r.y));
            const double t = 1.0 + cc * z;
            if (t <= 0.0) continue;
            const double v = t * t * t, u = u01(r.z);
            if (log(u) < 0.5 * z * z + dd - dd * v + dd * log(v)) {
                double g = dd * v;
                if (alpha < 1.0) g *= pow(u01(r.w), 1.0 / alpha);
                return g;
            }
        }
        return dd;
    }

    // player.py:395-428; returns the child rank (uniform)
    __device__ int select(const Node& nd, bool is_root) {
        const int nl = popc64(nd.legal);
        const Edge* ed = edges + nd.edge_base;
        Edge e0 = Edge{0, 0.f, 0.f, 0}, e1 = e0;
        if (lane < nl) e0 = ed[lane];
        if (lane + 32 < nl) e1 = ed[lane + 32];
        const int sum_n = __reduce_add_sync(kFull, e0.n + e1.n);
        const double xx = fmax(sqrt((double)sum_n), 1.0);
        const bool noisy = is_root && c.noise_eps > 0.f;
        double g0 = 0.0, g1 = 0.0, gsum = 0.0;
        if (noisy) {
            const uint32_t rootsel = sl.n_rootsel++;
            if (lane < nl) g0 = gamma_draw(rootsel, (uint32_t)lane);
            if (lane + 32 < nl) g1 = gamma_draw(rootsel, (uint32_t)lane + 32);
            for (int i = 0; i < nl; ++i)  // same left-to-right sum as the sequential kernel
                gsum += __shfl_sync(kFull, i < 32 ? g0 : g1, i & 31);
        }
        const float keep = (float)(1.0 - (double)c.noise_eps);
        const double eps = (double)c.noise_eps, cp = (double)c.c_puct;
        double bv = -1.0;
        int bi = 0x7fffffff;
#pragma unroll
        for (int half = 0; half < 2; ++half) {
            const int i = lane + 32 * half;
            if (i < nl) {
                const Edge& e = half ? e1 : e0;
                const double n = (double)e.n;
                double u;
                if (noisy) {
                    const float t32 = keep * e.p;
                    const double pr = (double)t32 + eps * ((half ? g1 : g0) / gsum);
                    u = cp * pr * xx / (1.0 + n);
                } else {
                    const float c32 = c.c_puct * e.p;
                    u = (double)c32 * xx / (1.0 + n);
                }
                const double q = (double)e.w / (n + 1e-5);
                const double v = q + u + 1000.0;
                if (v > bv) { bv = v; bi = i; }
            }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const double ov = __shfl_xor_sync(kFull, bv, o);
            const int oi = __shfl_xor_sync(kFull, bi, o);
            if (ov > bv || (ov == bv && oi < bi)) { bv = ov; bi = oi; }
        }
        return bi;
    }

    __device__ static int nth_set_bit(u64 m, int k) {
        for (int i = 0; i < k; ++i) m &= m - 1;
        return ctz64(m);
    }

    // ---- endgame solver hooks (agent/player.py:237-251); the WLD result of a position is cached in Node::pad:
    //      bit 15 solved, bit 6 has-move, bits 0-5 move, bits 7-8 sign(score) + 1
    __device__ static uint16_t wld_encode(int mv, int sc) {
        const int sg = sc > 0 ? 2 : (sc < 0 ? 0 : 1);
        return (uint16_t)(0x8000u | (mv >= 0 ? (0x40u | (uint32_t)mv) : 0u) | ((uint32_t)sg << 7));
    }
    // player.py:240-251 with the cached result; false when the reference's `if action:` fails (no move, or square 0)
    __device__ bool apply_wld(int ni, const uint32_t* path, int path_len, bool mover_is_root) {
        const Node nd = nodes[ni];
        const int action = nd.pad & 63;
        if (!(nd.pad & 0x40) || action == 0) return false;
        const float sgn = (float)(((nd.pad >> 7) & 3) - 1);   // value for the side to move at this node
        const int nl = popc64(nd.legal), r = popc64(nd.legal & ((1ULL << action) - 1));
        Edge* ed = edges + nd.edge_base;
        for (int i = lane; i < nl; i += 32) {
            Edge e = ed[i];
            e.p = i == r ? 1.f : 0.f;
            if (i == r) { e.n += 1; e.w = e.w + sgn; }
            ed[i] = e;
        }
        __syncwarp();
        backup(path, path_len, mover_is_root ? sgn : -sgn);
        return true;
    }

    // one simulation (oracle SelfPlayGame._run): 0 done, 1 pending (network), 2 parked, 3 pending (WLD solve)
    __device__ int run(int di) {
        Descent& D = desc[di];
        const int pid = sl.root_pid;
        u64 black = D.black, white = D.white;
        int np = D.next_player, path_len = D.path_len;
        const uint32_t kp = kpid_of(pid);
        while (true) {
            const bool black_to_move = np == 1;
            const u64 own = black_to_move ? black : white, enemy = black_to_move ? white : black;
            bool collide = false;
            for (int j = 0; j < sl.n_pending; ++j) {  // player.py:253-254
                const Descent& o = desc[sl.pending[j]];
                if (o.leaf_own == own && o.leaf_enemy == enemy) collide = true;
            }
            int ni = find_node(own, enemy, kp);
            if (c.solver_sim_turn > 0 && popc64(own | enemy) - 4 >= c.solver_sim_turn) {  // player.py:237-251
                if (ni >= 0 && (nodes[ni].pad & 0x8000)) {
                    __syncwarp();
                    if (apply_wld(ni, D.path, path_len, np == pid)) return 0;
                    // `if action:` failed: go on as if there were no solver
                } else if (!collide) {  // not solved yet: request the solve, the simulation waits for it like for the network
                    if (lane == 0) {
                        D.black = black; D.white = white; D.next_player = (uint8_t)np; D.path_len = (uint8_t)path_len;
                        D.dihedral = kSolveMarker;
                        D.leaf_own = own; D.leaf_enemy = enemy;
                        D.leaf_mover_is_root = (uint8_t)(np == pid);
                    }
                    __syncwarp();
                    return 3;
                }
            }
            if (collide) {
                if (lane == 0) { D.black = black; D.white = white; D.next_player = (uint8_t)np; D.path_len = (uint8_t)path_len; }
                __syncwarp();
                return 2;
            }
            if (ni < 0 || !((nodes[ni].exp >> (pid - 1)) & 1)) {  // player.py:257
                const U4 r = draw(c.seed, sl.game_id, sl.n_expand, P_DIHEDRAL, 0);
                const int flip = u01(r.x) < 0.5 ? 4 : 0;
                const int rot = (int)(u01(r.y) * 4.0);
                sl.n_expand++;
                if (lane == 0) {
                    D.black = black; D.white = white; D.next_player = (uint8_t)np; D.path_len = (uint8_t)path_len;
                    D.dihedral = (uint8_t)(flip | rot);
                    D.leaf_own = own; D.leaf_enemy = enemy;
                    D.leaf_mover_is_root = (uint8_t)(np == pid);
                }
                __syncwarp();
                return 1;
            }
            const Node nd = nodes[ni];
            const int r = select(nd, path_len == 0);
            if (path_len >= kMaxPath) { fail(RZ_ECAPACITY); return 0; }
            if (lane == 0) {
                Edge& e = edges[nd.edge_base + r];
                e.n += c.vl;  // player.py:270-271
                e.w = e.w - (float)c.vl;
                D.path[path_len] = (nd.edge_base + (uint32_t)r) | ((uint32_t)(np == pid) << 31);
            }
            ++path_len;
            const int a = nth_set_bit(nd.legal, r);
            const u64 fl = calc_flip(a, own, enemy);
            const u64 own2 = own ^ fl | (1ULL << a), en2 = enemy ^ fl;
            black = black_to_move ? own2 : en2;
            white = black_to_move ? en2 : own2;
            if (find_correct_moves(en2, own2)) np = black_to_move ? 2 : 1;
            else if (!find_correct_moves(own2, en2)) {  // game over: player.py:226-232
                const uint8_t w = winner_by_count(black, white);
                const float v = w == 3 ? 0.f : (w == pid ? 1.f : -1.f);
                __syncwarp();
                backup(D.path, path_len, v);
                return 0;
            }
            __syncwarp();
        }
    }

    // player.py:283-327 for one evaluated leaf
    __device__ void consume(int di) {
        const Descent& D = desc[di];
        const int pid = sl.root_pid;
        const uint32_t kp = kpid_of(pid);
        const u64 lown = D.leaf_own, lenemy = D.leaf_enemy;
        const int t = D.dihedral;
        int ni = find_node(lown, lenemy, kp);
        if (ni < 0) ni = create_node(lown, lenemy, kp);
        if (t == kSolveMarker) {  // result of a WLD solve requested in the previous wave
            sl.n_solves++;
            bool applied = false;
            if (ni >= 0) {
                const solver::SolveCtx& sc = p.sctx[(size_t)s * (c.K + 1) + di];
                if (lane == 0) nodes[ni].pad = wld_encode(sc.move, sc.score);
                __syncwarp();
                applied = apply_wld(ni, D.path, D.path_len, D.leaf_mover_is_root != 0);
            }
            if (applied || ni < 0) dstat[di] = D_FREE;
            else { dstat[di] = D_PARKED; sl.parked[sl.n_parked++] = (uint8_t)di; }  // continues from this node next wave
            return;
        }
        if (ni >= 0) {
            const Node nd = nodes[ni];
            const float* pol = D.kept ? p.keep_policy + ((size_t)s * c.K + di) * 64 : p.policy + (size_t)D.leaf_index * 64;
            const float a_lo = ((nd.legal >> lane) & 1ULL) ? pol[dihedral_square(lane, t)] : 0.f;
            const float a_hi = ((nd.legal >> (lane + 32)) & 1ULL) ? pol[dihedral_square(lane + 32, t)] : 0.f;
            // numpy float32 sum order: 8 running column sums over the rows, then a fixed tree
            const int j = lane & 7;
            float col = __shfl_sync(kFull, a_lo, j);
            col = col + __shfl_sync(kFull, a_lo, j + 8);
            col = col + __shfl_sync(kFull, a_lo, j + 16);
            col = col + __shfl_sync(kFull, a_lo, j + 24);
            col = col + __shfl_sync(kFull, a_hi, j);
            col = col + __shfl_sync(kFull, a_hi, j + 8);
            col = col + __shfl_sync(kFull, a_hi, j + 16);
            col = col + __shfl_sync(kFull, a_hi, j + 24);
            const float c0 = __shfl_sync(kFull, col, 0), c1 = __shfl_sync(kFull, col, 1), c2 = __shfl_sync(kFull, col, 2),
                        c3 = __shfl_sync(kFull, col, 3), c4 = __shfl_sync(kFull, col, 4), c5 = __shfl_sync(kFull, col, 5),
                        c6 = __shfl_sync(kFull, col, 6), c7 = __shfl_sync(kFull, col, 7);
            const float sum = ((c0 + c1) + (c2 + c3)) + ((c4 + c5) + (c6 + c7));
            const int nl = popc64(nd.legal);
            Edge* ed = edges + nd.edge_base;
            for (int i = lane; i < nl; i += 32) {
                const float v = pol[dihedral_square(nth_set_bit(nd.legal, i), t)];
                ed[i].p = sum > 0.f ? v / sum : v;
            }
            if (lane == 0) nodes[ni].exp = nd.exp | (uint8_t)(1u << (pid - 1));
            __syncwarp();
        }
        const float v = D.kept ? p.keep_value[(size_t)s * c.K + di] : p.value[D.leaf_index];
        backup(D.path, D.path_len, D.leaf_mover_is_root ? v : -v);
        if (D.kept && lane == 0) desc[di].kept = 0;
        dstat[di] = D_FREE;
    }

    __device__ void start_descent(int di) {
        if (lane == 0) {
            Descent& d = desc[di];
            const bool black_root = sl.root_pid == 1;
            d.black = black_root ? sl.root_own : sl.root_enemy;
            d.white = black_root ? sl.root_enemy : sl.root_own;
            d.next_player = sl.root_pid;
            d.path_len = 0;
        }
        __syncwarp();
    }

    __device__ bool search_wave() {
        while (true) {
            uint8_t still[kMaxK];
            int n_still = 0;
            int started_wave = 0;
            sl.n_pending = 0;
            for (int j = 0; j < sl.n_parked; ++j) {
                const int di = sl.parked[j];
                const int r = run(di);
                if (r == 2) still[n_still++] = (uint8_t)di;
                else if (r == 1 || r == 3) { dstat[di] = D_PENDING; sl.pending[sl.n_pending++] = (uint8_t)di; }
                else dstat[di] = D_FREE;
            }
            while (sl.sims_started < sl.sims_target && sl.n_pending + n_still < c.K && started_wave < c.sims_cap) {
                int di = 0;
                ++started_wave;
                while (dstat[di] != D_FREE) ++di;
                sl.sims_started++;
                start_descent(di);
                dstat[di] = D_PARKED;
                const int r = run(di);
                if (r == 2) still[n_still++] = (uint8_t)di;
                else if (r == 1 || r == 3) { dstat[di] = D_PENDING; sl.pending[sl.n_pending++] = (uint8_t)di; }
                else dstat[di] = D_FREE;
            }
            sl.n_parked = (uint8_t)n_still;
            for (int j = 0; j < n_still; ++j) sl.parked[j] = still[j];
            if (sl.n_pending > 0) return true;
            if (sl.sims_started >= sl.sims_target) return false;
            return true;  // cap reached with nothing to evaluate: continue in the next wave
        }
    }

    __device__ void begin_search(u64 own, u64 enemy, int pid) {
        sl.root_own = own; sl.root_enemy = enemy; sl.root_pid = (uint8_t)pid;
        sl.sims_started = 0; sl.sims_target = (uint32_t)c.S;
        sl.n_pending = 0; sl.n_parked = 0;
        sl.phase = PH_SEARCH;
    }

    // start of a ply (agent/player.py:95-109): from use_solver_turn on, ask the exact solver first (:100-103)
    __device__ void begin_ply(u64 own, u64 enemy, int pid) {
        if (c.solver_turn > 0 && popc64(own | enemy) - 4 >= c.solver_turn) {
            sl.root_own = own; sl.root_enemy = enemy; sl.root_pid = (uint8_t)pid;
            sl.root_req = 1;
            sl.phase = PH_SOLVE;
            return;
        }
        begin_search(own, enemy, pid);
    }

    // action_by_searching, agent/player.py:150-161, with the result of the exact solve requested in the previous wave
    __device__ void consume_root_solve() {
        const u64 own = sl.root_own, enemy = sl.root_enemy;
        const int pid = sl.root_pid;
        const solver::SolveCtx& rc = p.sctx[(size_t)s * (c.K + 1) + c.K];
        const int mv = rc.move, sc = rc.score;
        sl.n_solves++;
        if (mv < 0) { begin_search(own, enemy, pid); return; }  // refused (the reference: timeout) -> search as usual
        const uint32_t kp = kpid_of(pid);
        int ni = find_node(own, enemy, kp);
        if (ni < 0) ni = create_node(own, enemy, kp);
        if (ni < 0) { sl.phase = PH_IDLE; return; }
        const Node nd = nodes[ni];
        const float sgn = sc > 0 ? 1.f : (sc < 0 ? -1.f : 0.f);
        const int nl = popc64(nd.legal), r = popc64(nd.legal & ((1ULL << mv) - 1));
        Edge* ed = edges + nd.edge_base;
        for (int i = lane; i < nl; i += 32) {
            Edge e = ed[i];
            e.p = i == r ? 1.f : 0.f;
            if (i == r) { e.n = 999; e.w = sgn * 999.f; }
            ed[i] = e;
        }
        __syncwarp();
        if ((int)sl.ply >= c.max_plies) { fail(RZ_ECAPACITY); sl.phase = PH_IDLE; return; }
        rz_ply& pl = p.plies[((size_t)s * 2 + sl.log_sel) * c.max_plies + sl.ply];
        for (int sq = lane; sq < 64; sq += 32)
            pl.n_visit[sq] = ((nd.legal >> sq) & 1ULL) ? ed[popc64(nd.legal & ((1ULL << sq) - 1))].n : 0;
        if (lane == 0) {
            pl.own = own; pl.enemy = enemy;
            pl.player = (uint8_t)pid; pl.loops = 0; pl.pad = 0;
            pl.waves = (uint16_t)(sl.ply_waves > 0xFFFFu ? 0xFFFFu : sl.ply_waves);
            pl.n = 999.f; pl.q = sgn;
            pl.action = (int16_t)mv;
            pl.recorded = 0;  // "not save move as play data", player.py:102
            atomicAdd(&p.status->plies, 1ULL);
        }
        __syncwarp();
        sl.ply++;
        sl.ply_waves = 0;
        env_step(sl.env, mv);
        if (sl.env.done) { finish_game(); return; }
        const bool b2 = sl.env.next_player == 1;
        begin_ply(b2 ? sl.env.black : sl.env.white, b2 ? sl.env.white : sl.env.black, sl.env.next_player);
    }

    // rz_engine_set_openings (max_games bounds `local` by the table's length): the opening's plies are played without a
    // search and not recorded; the host checked that none passes or ends the game.  Kept out of line: inlined into the
    // tick kernel it costs new_game's callers registers.
    __device__ __noinline__ void play_opening(u64 local) {
        const uint8_t* op = p.openings + local * kOpeningStride;
        sl.opening_plies = op[0];
        for (int i = 0; i < (int)sl.opening_plies; ++i) env_step(sl.env, op[1 + i]);
        if (sl.opening_plies) {
            const bool b = sl.env.next_player == 1;
            begin_ply(b ? sl.env.black : sl.env.white, b ? sl.env.white : sl.env.black, sl.env.next_player);
        }
    }

    __device__ void new_game() {
        const u64 local = (u64)s + sl.games_played * (u64)c.G;
        if (c.max_games && local >= c.max_games) {
            sl.phase = PH_IDLE;
            if (lane == 0) atomicAdd(&p.status->idle_slots, 1ULL);
            return;
        }
        sl.game_id = c.first_game_id + local * c.game_id_stride;
        if (p.net_table) {  // rz_engine_set_nets (max_games bounds `local` by the table's length)
            sl.black_net = p.net_table[2 * local];
            sl.white_net = p.net_table[2 * local + 1];
        } else {  // self-play: network 0; two networks without a table: colours alternate with the game
            sl.black_net = c.n_nets > 1 ? (uint8_t)(local & 1) : (uint8_t)0;
            sl.white_net = c.n_nets > 1 ? (uint8_t)(1 - sl.black_net) : (uint8_t)0;
        }
        sl.games_played++;
        env_reset(sl.env);
        if (c.keep_games > 1 && (sl.games_played - 1) % (u64)c.keep_games != 0) {
            // reset_mtcs_info_per_game > 1 (worker/self_play.py:111-134): the statistics of the previous game stay; the two
            // new players regard every position that has a prior as expanded (player.py:47 expanded = set(var_p.keys()))
            for (uint32_t i = lane; i < sl.n_nodes; i += 32) nodes[i].exp = 3;
            __syncwarp();
        } else {
            sl.gen = sl.gen + 1;
            if (sl.gen >= 4096) {
                for (uint32_t i = lane; i < c.hash_cap; i += 32) hash[i] = 0;
                sl.gen = 1;
                __syncwarp();
            }
            sl.n_nodes = 0; sl.n_edges = 0;
        }
        sl.n_expand = 0; sl.n_rootsel = 0; sl.n_sims = 0; sl.ply = 0; sl.tl = 0;
        sl.n_searched_plies = 0; sl.n_solves = 0; sl.root_req = 0;
        sl.resigned_mask = 0; sl.search_only = 0; sl.ply_waves = 0;
        for (int k = 0; k < c.K; ++k) dstat[k] = D_FREE;
        sl.enable_resign = (uint8_t)((double)c.disable_resignation_rate <= u01(draw(c.seed, sl.game_id, 0, P_GAME, 0).x));
        if (lane == 0) atomicAdd(&p.status->games_started, 1ULL);
        sl.phase = PH_DECIDE;
        sl.opening_plies = 0;
        if (p.openings) play_opening(local);
        if (c.warm_start && sl.games_played == 1) {
            // the slot's first game starts at turn `pre` (drawn from the profile, rz_engine_set_warm_start_profile) after
            // `pre` random legal plies, and its first search is a uniformly drawn part of a whole one: the state of a slot
            // met at a random moment of a long run.  Pre-played plies are neither searched nor recorded.
            const U4 r0 = draw(c.seed, sl.game_id, 1, P_GAME, 0);
            const float u = (float)u01(r0.x);
            int pre = 0;
            while (pre < 59 && u >= c.warm_cdf[pre]) ++pre;
            // a random playout that ends before turn `pre` is drawn again (another stream), so that late turns are not
            // under-represented; after 8 failures the slot starts a fresh game
            for (uint32_t attempt = 0; attempt < 8; ++attempt) {
                env_reset(sl.env);
                for (int i = 0; i < pre && !sl.env.done; ++i) {
                    const bool b = sl.env.next_player == 1;
                    const u64 legal = find_correct_moves(b ? sl.env.black : sl.env.white, b ? sl.env.white : sl.env.black);
                    const U4 r = draw(c.seed, sl.game_id, 2 + (uint32_t)i + 64u * attempt, P_GAME, 0);
                    env_step(sl.env, nth_set_bit(legal, (int)(u01(r.x) * (double)popc64(legal))));
                }
                if (!sl.env.done) break;
            }
            if (sl.env.done) env_reset(sl.env);
            else if (sl.env.turn > 0) {
                const bool b = sl.env.next_player == 1;
                begin_ply(b ? sl.env.black : sl.env.white, b ? sl.env.white : sl.env.black, sl.env.next_player);
                if (sl.phase == PH_SEARCH) {
                    // The first search runs a uniformly drawn part of a whole one.  Late in the game a search of a long-running
                    // engine is short in WAVES (its simulations end in terminal positions already in the tree: 24 instead of 50
                    // waves at 400 simulations), while this slot's tree is empty and needs the network for every simulation, K per
                    // wave: the part is drawn from the waves the profile gives the turn, so that the slot decides when its
                    // steady-state twin would.  At least two simulations: the first one only expands the root.
                    const double whole = (c.warm_waves[pre] > 0.f && (double)c.warm_waves[pre] * c.K < (double)c.S) ? (double)c.warm_waves[pre] * c.K
                                                                                                               : (double)c.S;
                    uint32_t part = (uint32_t)(u01(r0.y) * whole) + 1u;
                    if (part < 2u) part = 2u;
                    sl.sims_target = part < (uint32_t)c.S ? part : (uint32_t)c.S;
                }
            }
        }
    }

    __device__ void finish_game() {
        if (lane == 0) {
            rz_game& g = p.mail_hdr[(size_t)s * 2 + sl.log_sel];
            g.game_id = sl.game_id; g.black = sl.env.black; g.white = sl.env.white;
            g.first_ply = 0; g.n_plies = (int32_t)sl.ply; g.expansions = (int32_t)sl.n_expand; g.simulations = (int32_t)sl.n_sims;
            g.winner = sl.env.winner; g.black_z = sl.env.winner == 1 ? 1 : (sl.env.winner == 2 ? -1 : 0);
            g.resign_enabled = sl.enable_resign; g.resigned_mask = sl.resigned_mask; g.turn = sl.env.turn;
            g.black_net = sl.black_net; g.white_net = sl.white_net; g.opening_plies = sl.opening_plies;
            g.table_nodes = (int32_t)sl.n_nodes; g.pad2 = 0;
            atomicMax(&p.status->max_nodes, (unsigned long long)sl.n_nodes);
            atomicMax(&p.status->max_edges, (unsigned long long)sl.n_edges);
            __threadfence();
            p.mail_flag[(size_t)s * 2 + sl.log_sel] = 1;
            atomicAdd(&p.status->games_finished, 1ULL);
        }
        __syncwarp();
        sl.log_sel ^= 1;
        sl.phase = PH_NEWGAME;
    }

    // player.py:82-134 + self_play.py:155-162 (same statements as Ctx::decide; stores by lane 0)
    __device__ void decide() {
        const bool black_to_move = sl.env.next_player == 1;
        const int pid = sl.env.next_player;
        const u64 own = black_to_move ? sl.env.black : sl.env.white, enemy = black_to_move ? sl.env.white : sl.env.black;
        const int turn = popc64(own) + popc64(enemy) - 4;
        const uint32_t kp = kpid_of(pid);
        int ni = find_node(own, enemy, kp);
        if (turn == 0) {  // bypass_first_move
            if (ni < 0) ni = create_node(own, enemy, kp);
            if (ni < 0) { sl.phase = PH_IDLE; return; }
            const Node nd0 = nodes[ni];
            const int nl0 = popc64(nd0.legal);
            Edge* ed0 = edges + nd0.edge_base;
            for (int i = lane; i < nl0; i += 32) {
                Edge e = ed0[i];
                if (i == 0) { e.n = 1; e.w = 0.f; }
                e.p = 1.0f / (float)nl0;
                ed0[i] = e;
            }
            __syncwarp();
        }
        if (ni < 0) { fail(RZ_ESTATE); sl.phase = PH_IDLE; return; }
        const Node nd = nodes[ni];
        const int nl = popc64(nd.legal);
        const Edge* ed = edges + nd.edge_base;
        long long sum_n = 0;
        int arg_n = 0;
        for (int i = 0; i < nl; ++i) { sum_n += ed[i].n; if (ed[i].n > ed[arg_n].n) arg_n = i; }
        const bool tau1 = turn < c.change_tau_turn;
        const U4 r = draw(c.seed, sl.game_id, sl.n_searched_plies * 16 + sl.tl, P_MOVE, 0);
        const double uu = u53(r.x, r.y);
        int choice = arg_n;
        if (tau1) {
            double total = 0.0;
            for (int i = 0; i < nl; ++i) total += (double)ed[i].n / (double)sum_n;
            double cum = 0.0;
            choice = nl - 1;
            for (int i = 0; i < nl; ++i) {
                cum += (double)ed[i].n / (double)sum_n;
                if (cum / total > uu) { choice = i; break; }
            }
        }
        int abv = -1;
        double q_abv = 0.0, max_q_visited = -10.0;
        for (int i = 0; i < nl; ++i) {
            if (ed[i].n > 0) {
                const double q = (double)ed[i].w / ((double)ed[i].n + 1e-5);
                if (abv < 0 || q + 100.0 > q_abv + 100.0) { abv = i; q_abv = q; }
                if (q > max_q_visited) max_q_visited = q;
            }
        }
        const double q_choice = (double)ed[choice].w / ((double)ed[choice].n + 1e-5);
        const double value_diff = q_choice - q_abv;
        sl.tl++;
        const bool accept = turn <= c.start_rethinking_turn || (value_diff > -0.01 && ed[choice].n >= c.required_visit);
        const bool room = (u64)sl.n_nodes + (u64)c.S * (u64)(61 - turn) + 64 <= (u64)c.nodes_cap;
        if (!accept && sl.tl < c.thinking_loop && turn > 0 && room) {
            begin_search(own, enemy, pid);
            return;
        }
        const int action = nth_set_bit(nd.legal, choice);
        if ((int)sl.ply >= c.max_plies) { fail(RZ_ECAPACITY); sl.phase = PH_IDLE; return; }
        rz_ply& pl = p.plies[((size_t)s * 2 + sl.log_sel) * c.max_plies + sl.ply];
        bool resign = false;
        if (c.use_resign && max_q_visited <= (double)c.resign_threshold) {
            sl.resigned_mask |= (uint8_t)(1u << (pid - 1));
            if (sl.enable_resign && turn >= c.allowed_resign_turn) resign = true;
        }
        for (int sq = lane; sq < 64; sq += 32)
            pl.n_visit[sq] = ((nd.legal >> sq) & 1ULL) ? ed[popc64(nd.legal & ((1ULL << sq) - 1))].n : 0;
        if (lane == 0) {
            pl.own = own; pl.enemy = enemy;
            pl.player = (uint8_t)pid; pl.loops = sl.tl; pl.pad = 0;
            pl.waves = (uint16_t)(sl.ply_waves > 0xFFFFu ? 0xFFFFu : sl.ply_waves);
            pl.n = (float)ed[choice].n; pl.q = (float)q_choice;
            pl.action = resign ? (int16_t)-1 : (int16_t)action;
            pl.recorded = resign ? 0 : 1;
            atomicAdd(&p.status->plies, 1ULL);
        }
        __syncwarp();
        sl.ply++;
        sl.ply_waves = 0;
        sl.n_searched_plies++;
        sl.tl = 0;
        env_step(sl.env, resign ? -1 : action);
        if (sl.env.done) { finish_game(); return; }
        const bool b2 = sl.env.next_player == 1;
        begin_ply(b2 ? sl.env.black : sl.env.white, b2 ? sl.env.white : sl.env.black, sl.env.next_player);
    }
};

constexpr int kWarpTickThreads = 64;  // 2 game slots per CTA

__global__ void __launch_bounds__(kWarpTickThreads) tick_warp_kernel(const DevCfg c, const DevPtrs p, const int slot0, const int slot_end,
                                                                     const int group, const int parity) {
    const int lane = threadIdx.x & 31;
    const int s = slot0 + (int)((blockIdx.x * blockDim.x + threadIdx.x) >> 5);
    if (s >= slot_end) return;  // whole warps only
    if (p.status->error != 0) return;
    WCtx x(c, p, s, lane);
    Slot& sl = x.sl;
    if (sl.phase == PH_IDLE) return;
    if (sl.phase == PH_SEARCH || sl.phase == PH_SOLVE) sl.ply_waves++;
    if (sl.phase == PH_SEARCH) {  // 1. consume the previous wave's evaluations in request order
        // ... once every endgame solve the slot asked for is finished: a solve may take several waves, and until then the
        // slot does nothing (the search result cannot depend on how long a solve took).  Network results that arrived in
        // the meantime are copied out of the batch buffers, which the next wave overwrites.
        bool ready = true;
        for (int j = 0; j < (int)sl.n_pending; ++j) {
            const int di = sl.pending[j];
            if (x.desc[di].dihedral == kSolveMarker && !p.sctx[(size_t)s * (c.K + 1) + di].done) ready = false;
        }
        if (!ready) {
            for (int j = 0; j < (int)sl.n_pending; ++j) {
                const int di = sl.pending[j];
                Descent& d = x.desc[di];
                if (d.dihedral == kSolveMarker || d.kept) continue;
                float* kp = p.keep_policy + ((size_t)s * c.K + di) * 64;
                const float* src = p.policy + (size_t)d.leaf_index * 64;
                kp[lane] = src[lane]; kp[lane + 32] = src[lane + 32];
                if (lane == 0) { p.keep_value[(size_t)s * c.K + di] = p.value[d.leaf_index]; }
                __syncwarp();
                if (lane == 0) d.kept = 1;
            }
            __syncwarp();
            return;
        }
        const uint32_t consumed = sl.n_pending;
        uint32_t nn_consumed = 0;
        for (int j = 0; j < (int)consumed; ++j) {
            nn_consumed += x.desc[sl.pending[j]].dihedral != kSolveMarker;
            x.consume(sl.pending[j]);
        }
        sl.n_pending = 0;
        if (nn_consumed && lane == 0) atomicAdd(&p.status->expansions, (unsigned long long)nn_consumed);
    } else if (sl.phase == PH_SOLVE && !sl.root_req) {
        if (!p.sctx[(size_t)s * (c.K + 1) + c.K].done) return;  // the exact root solve needs more waves
        x.consume_root_solve();
    }
    for (int guard = 0; guard < 100000; ++guard) {  // 2. advance the state machine until the network is needed
        if (p.status->error != 0) break;
        if (sl.phase == PH_SEARCH) {
            if (x.search_wave()) break;
            sl.n_sims += sl.sims_started;
            if (lane == 0) atomicAdd(&p.status->simulations, (unsigned long long)sl.sims_started);
            if (sl.search_only) { sl.phase = PH_IDLE; if (lane == 0) atomicAdd(&p.status->idle_slots, 1ULL); break; }
            sl.phase = PH_DECIDE;
        } else if (sl.phase == PH_DECIDE) {
            x.decide();
        } else if (sl.phase == PH_NEWGAME) {
            if (p.mail_flag[(size_t)s * 2 + sl.log_sel]) break;
            x.new_game();
        } else {
            break;  // PH_SOLVE: the exact root solve is requested below and consumed in the next wave
        }
    }
    const int n_leaves = sl.phase == PH_SEARCH ? sl.n_pending : 0;
    const uint32_t root_req = (sl.phase == PH_SOLVE && sl.root_req) ? 1u : 0u;
    // 3. gather: network leaves (K3: dihedral-transformed bitboards) and solver requests go to their own compact batches
    const bool mine = lane < n_leaves;
    const bool is_solve = mine && x.desc[sl.pending[mine ? lane : 0]].dihedral == kSolveMarker;
    const bool is_leaf = mine && !is_solve;
    u64 t_own = 0, t_enemy = 0;
    bool hit = false;
    if (is_leaf) {
        const Descent& d = x.desc[sl.pending[lane]];
        t_own = dihedral(d.leaf_own, d.dihedral);
        t_enemy = dihedral(d.leaf_enemy, d.dihedral);
        if (p.cache.n_sets) {  // a hit goes to the descent's keep row, which consume() reads when `kept` is set
            const size_t row = (size_t)s * c.K + sl.pending[lane];
            hit = cache_lookup(p.cache, t_own, t_enemy, p.keep_policy + row * 64, p.keep_value + row);
        }
    }
    const unsigned sv_mask = __ballot_sync(0xffffffffu, is_solve), nn_mask = __ballot_sync(0xffffffffu, is_leaf && !hit);
    const uint32_t n_nn = __popc(nn_mask), n_sv = __popc(sv_mask) + root_req;
    const uint32_t n_hit = __popc(__ballot_sync(0xffffffffu, hit));
    if (lane == 0 && n_nn + n_hit > 0) {
        if (p.cache.n_sets) {
            const int turn = popc64(sl.root_own | sl.root_enemy) - 4;
            const int b = (c.warm_start && sl.games_played == 1) ? kCacheTurnBuckets - 1 : (turn < 0 ? 0 : (turn > 59 ? 59 : turn));
            atomicAdd(&p.status->cache_lookups[b], (unsigned long long)(n_nn + n_hit));
            if (n_hit) atomicAdd(&p.status->cache_hits[b], (unsigned long long)n_hit);
        }
        if (n_nn) atomicAdd(&p.status->tower_rows, (unsigned long long)n_nn);
    }
    const uint32_t net = sl.root_pid == 1 ? sl.black_net : sl.white_net;  // the searching player's network (0 in self-play)
    uint32_t base = 0, sbase = 0;
    uint32_t* s_count = p.solve_count + (group * 2 + parity) * 64;
    uint32_t* s_list = p.sactive + (size_t)(group * 2 + parity) * c.G * (c.K + 1);
    if (lane == 0 && n_nn > 0) base = atomicAdd(p.batch_count + (group * c.n_nets + net) * 64, n_nn);
    if (lane == 0 && n_sv > 0) sbase = atomicAdd(s_count, n_sv);
    base = __shfl_sync(0xffffffffu, base, 0);
    sbase = __shfl_sync(0xffffffffu, sbase, 0);
    if (root_req) sl.root_req = 0;
    x.write_back();
    const uint32_t below = (1u << lane) - 1u;
    if (hit) {
        x.desc[sl.pending[lane]].kept = 1;
    } else if (is_leaf) {
        Descent& d = x.desc[sl.pending[lane]];
        const uint32_t at = net * (uint32_t)c.G * (uint32_t)c.K + (uint32_t)slot0 * (uint32_t)c.K + base + __popc(nn_mask & below);
        d.leaf_index = at;
        d.kept = 0;
        p.batch_own[at] = t_own;
        p.batch_enemy[at] = t_enemy;
    } else if (is_solve) {  // WLD solve of a simulation's position: context of this descent
        const int di = sl.pending[lane];
        const Descent& d = x.desc[di];
        const uint32_t idx = (uint32_t)s * (uint32_t)(c.K + 1) + (uint32_t)di;
        solver::ctx_init(p.sctx + idx, d.leaf_own, d.leaf_enemy, 0);
        s_list[sbase + __popc(sv_mask & below)] = idx;
    }
    if (root_req && lane == 0) {  // exact solve of the root: the slot's own context
        const uint32_t idx = (uint32_t)s * (uint32_t)(c.K + 1) + (uint32_t)c.K;
        solver::ctx_init(p.sctx + idx, sl.root_own, sl.root_enemy, 1);
        s_list[sbase + (n_sv - 1)] = idx;
    }
}
