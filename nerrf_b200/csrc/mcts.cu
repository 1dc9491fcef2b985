// planner.mcts.search + planner.rewards.score (SURVEY.md 8a rows a5, a6; DESIGN.md "MCTS spec").
//
// Bit-exact restatement of oracle/mcts_ref.py + oracle/rewards_ref.py: integer visit counts and
// action indices, Philox4x32-10 counter RNG, and fp32 arithmetic written with explicitly rounded
// intrinsics (__fadd_rn / __fmul_rn / __fdiv_rn / __fsqrt_rn: never contracted to FMA) in the
// spec'd association order.
//
// One PERSISTENT cooperative kernel runs all T iterations of the leaf-parallel search:
//   select   every CTA redundantly descends the tree (block-wide UCT argmax per level; tree is
//            L2-resident and read with ld.global.cg) -> no grid barrier between select/rollout
//   rollout  one warp per rollout: lane l holds NW 32-bit words of the action bitset; j-th
//            legal action = warp prefix-sum of popcounts + __fns; reward = per-lane sequential
//            sum over its 32*NW actions (terms staged in smem, transposed -> conflict-free)
//            + xor-butterfly; value written to val[r]
//   grid barrier (monotonic counter: one atomicAdd + ld.acquire spin per CTA; co-residency is guaranteed by
//                 the cooperative launch; cheaper than cg::grid.sync with one fat CTA per SM) -- the ONLY one per
//                 iteration: every CTA keeps its own replica of the tree and applies the (deterministic) backup to it
//                 redundantly from the shared rollout values, so no CTA ever waits for another CTA's tree writes;
//                 val[] is double buffered across iterations
//   backup   every CTA, on its replica: adjacent-pairs tree sum of val -> path edges; per-first-action child
//            statistics of the leaf (fixed ascending-r order)
// Reward spec v1 (oracle/rewards_ref.py): an applied action whose GUARD (a "kill process" action, index < 32, i.e. a
// bit of state word 0) is not applied contributes vw_a = fl(v_a + fl(p_g * u_a)) instead of v_a.
// Reward spec v2 (oracle/restore_ref.py): an action may also name a COVER -- the "restore from snapshot" action (index
// < 32, state word 0) of its directory.  An action that is not applied but whose cover is applied is restored all the
// same: its data-loss term is v_a (vw_a while its guard lives) and its downtime term is 0.
#include "common.cuh"

#include <vector>

namespace nerrf {

constexpr int MAXD = 256;
constexpr int MCTS_THREADS = 896;     // 28 warps, one CTA per SM (72 registers: 896 threads fill the register file)
constexpr int MCTS_WARPS = MCTS_THREADS / 32;
constexpr int MAXR = 8192;

__device__ __forceinline__ void philox4x32_10(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3, uint32_t k0,
                                              uint32_t k1, uint32_t out[4]) {
    constexpr uint32_t M0 = 0xD2511F53u, M1 = 0xCD9E8D57u, W0 = 0x9E3779B9u, W1 = 0xBB67AE85u;
#pragma unroll
    for (int r = 0; r < 10; ++r) {
        const uint32_t hi0 = __umulhi(M0, c0), lo0 = M0 * c0;
        const uint32_t hi1 = __umulhi(M1, c2), lo1 = M1 * c2;
        const uint32_t n0 = hi1 ^ c1 ^ k0, n2 = hi0 ^ c3 ^ k1;
        c0 = n0; c1 = lo1; c2 = n2; c3 = lo0;
        k0 += W0; k1 += W1;
    }
    out[0] = c0; out[1] = c1; out[2] = c2; out[3] = c3;
}

// Staged reward terms, transposed (action a = lane*chunk + i lives at [i*32 + lane]): three tables of (data-loss term,
// downtime term) PAIRS -- tab[0] = (u, 0) for an action that is NOT applied, tab[1] = (v, cost) applied, tab[2] = (vw, cost)
// applied while its guard (kill) action is not -- so evaluating one action is one 8-byte shared load from the table the
// state selects, + two rounded adds (r1/r2: five loads and three selects per action, ~600 instructions per state).
// Spec v2 (covers) adds two more tables -- ctab[0] = (v, 0) restored by its cover, ctab[1] = (vw, 0) restored while its
// guard lives -- and the cover byte table.  They live in a separate region the caller places AFTER everything else the
// kernel keeps in dynamic shared memory, and are only allocated when covers are passed: without covers every offset, the
// shared-memory size and the occupancy are what they were in spec v1.
struct TermsS { float2* tab; uint8_t* g; bool has_guard; float2* ctab; uint8_t* cv; bool has_cover; };
template <int NW>
__device__ __forceinline__ TermsS carve_terms(unsigned char* smem, unsigned char* cover_smem) {
    constexpr int A_PAD = 1024 * NW;
    TermsS t;
    t.tab = reinterpret_cast<float2*>(smem);
    t.g = reinterpret_cast<uint8_t*>(t.tab + 3 * A_PAD);
    t.has_guard = false;
    t.ctab = reinterpret_cast<float2*>(cover_smem);
    t.cv = reinterpret_cast<uint8_t*>(t.ctab + 2 * A_PAD);
    t.has_cover = false;
    return t;
}
template <int NW>
constexpr size_t terms_smem_bytes() { return (size_t)1024 * NW * (3 * 8 + 1); }
// the cover region (spec v2), appended only when covers are passed
template <int NW>
constexpr size_t cover_smem_bytes() { return (size_t)1024 * NW * (2 * 8 + 1); }
// the search kernel appends one scratch bitset (32*NW words) per warp: the rank-space rollouts scatter their picks into it
template <int NW>
constexpr size_t mcts_smem_bytes() { return terms_smem_bytes<NW>() + (size_t)(896 / 32) * 32 * NW * 4; }

// block-wide (contains __syncthreads): fills the tables and reports whether any action has a guard / a cover.  `cover` is
// non-null only when the cover region was allocated.
template <int NW>
__device__ __forceinline__ void stage_terms(const float* __restrict__ p, const float* __restrict__ size,
                                            const float* __restrict__ cost, const int32_t* __restrict__ guard,
                                            const int32_t* __restrict__ cover, int A, TermsS& t) {
    constexpr int CHUNK = 32 * NW, A_PAD = 1024 * NW;
    int any = 0, any_cover = 0;
    for (int a = threadIdx.x; a < A_PAD; a += blockDim.x) {
        float u = 0.f, v = 0.f, vw = 0.f, c = 0.f;
        int g = 255;
        if (a < A) {
            const float pa = p[a], sa = size[a];
            u = __fmul_rn(pa, sa);
            v = __fmul_rn(__fsub_rn(1.0f, pa), sa);
            c = cost[a];
            vw = v;
            const int gd = guard ? guard[a] : -1;
            if (gd >= 0 && gd < 32 && gd < A) { g = gd; vw = __fadd_rn(v, __fmul_rn(p[gd], u)); any = 1; }
        }
        const int lane = a / CHUNK, i = a % CHUNK;
        t.tab[i * 32 + lane] = make_float2(u, 0.f);
        t.tab[A_PAD + i * 32 + lane] = make_float2(v, c);
        t.tab[2 * A_PAD + i * 32 + lane] = make_float2(vw, c);
        t.g[i * 32 + lane] = (uint8_t)g;
        if (cover) {                                                      // (uniform) spec v2
            const int cd = a < A ? cover[a] : -1;
            const bool on = cd >= 0 && cd < 32 && cd < A;
            any_cover |= on ? 1 : 0;
            t.ctab[i * 32 + lane] = make_float2(v, 0.f);
            t.ctab[A_PAD + i * 32 + lane] = make_float2(vw, 0.f);
            t.cv[i * 32 + lane] = (uint8_t)(on ? cd : 255);
        }
    }
    t.has_guard = __syncthreads_or(any) != 0;
    if (cover) t.has_cover = __syncthreads_or(any_cover) != 0;
}

// score of the state held across a warp (lane holds words w[0..NW)), spec'd order.  All lanes return it.
template <int NW>
__device__ __forceinline__ float warp_score(const uint32_t (&w)[NW], const TermsS t, int lane) {
    constexpr int A_PAD = 1024 * NW;
    float dl = 0.f, dt = 0.f;
    const float2* tab = t.tab + lane;
    if (t.has_cover) {                                                    // (uniform) spec v2: guards and covers
        const uint32_t w0 = __shfl_sync(0xffffffffu, w[0], 0);          // state word 0 holds the kill and restore actions
        const float2* ctab = t.ctab + lane;
#pragma unroll
        for (int k = 0; k < NW; ++k) {
#pragma unroll 8
            for (int b = 0; b < 32; ++b) {
                const int i = k * 32 + b;
                const unsigned ap = (w[k] >> b) & 1u;
                const unsigned gd = t.g[i * 32 + lane], cd = t.cv[i * 32 + lane];
                const unsigned guard_alive = (gd < 32u && !((w0 >> (gd & 31u)) & 1u)) ? 1u : 0u;
                const bool covered = cd < 32u && ((w0 >> (cd & 31u)) & 1u);
                // applied: (v|vw, cost); restored by its cover only: (v|vw, 0); neither: (u, 0)
                const float2* src = ap ? tab + (1u + guard_alive) * A_PAD : (covered ? ctab + guard_alive * A_PAD : tab);
                const float2 e = src[i * 32];
                dl = __fadd_rn(dl, e.x);
                dt = __fadd_rn(dt, e.y);
            }
        }
    } else if (!t.has_guard) {                                                   // (uniform) no guards: two tables
#pragma unroll
        for (int k = 0; k < NW; ++k) {
#pragma unroll 8
            for (int b = 0; b < 32; ++b) {
                const int i = k * 32 + b;
                const float2 e = tab[((w[k] >> b) & 1u) * A_PAD + i * 32];
                dl = __fadd_rn(dl, e.x);
                dt = __fadd_rn(dt, e.y);
            }
        }
    } else {
        const uint32_t w0 = __shfl_sync(0xffffffffu, w[0], 0);          // state word 0 holds the guard (kill) actions
#pragma unroll
        for (int k = 0; k < NW; ++k) {
#pragma unroll 8
            for (int b = 0; b < 32; ++b) {
                const int i = k * 32 + b;
                const unsigned ap = (w[k] >> b) & 1u;
                const unsigned gd = t.g[i * 32 + lane];
                const unsigned guard_alive = (gd < 32u && !((w0 >> (gd & 31u)) & 1u)) ? 1u : 0u;
                const float2 e = tab[(ap + (ap & guard_alive)) * A_PAD + i * 32];
                dl = __fadd_rn(dl, e.x);
                dt = __fadd_rn(dt, e.y);
            }
        }
    }
#pragma unroll
    for (int s = 1; s < 32; s <<= 1) {
        dl = __fadd_rn(dl, __shfl_xor_sync(0xffffffffu, dl, s));
        dt = __fadd_rn(dt, __shfl_xor_sync(0xffffffffu, dt, s));
    }
    return -__fadd_rn(dl, __fmul_rn(0.1f, dt));
}

// apply the j-th legal (zero) action, ascending a, to the warp-distributed state.  zl = this lane's
// zero count, incl = inclusive prefix over lanes; both are UPDATED in place (the chosen lane loses one
// zero, so every prefix from that lane on drops by one): no re-scan for the next step.
// The n-th-set-bit search inside the chosen word is done by the whole warp: the word is broadcast,
// lane b tests "bit b is legal and exactly `rank` legal bits lie below it", one ballot finds b.
template <int NW>
__device__ __forceinline__ void apply_jth(uint32_t (&w)[NW], int& zl, int& incl, int j, int lane) {
    const unsigned m = __ballot_sync(0xffffffffu, incl > j);
    const int src = __ffs(m) - 1;
    int rank = j - (incl - zl);                       // meaningful in lane `src` only
    int kk = 0;
    uint32_t zsel = ~w[0];
#pragma unroll
    for (int k = 1; k < NW; ++k) {                    // pick the word that holds the rank-th legal bit of this lane
        const int pz = __popc(zsel);
        const bool next = (kk == k - 1) && (rank >= pz);
        if (next) { rank -= pz; kk = k; zsel = ~w[k]; }
    }
    const uint32_t z = __shfl_sync(0xffffffffu, zsel, src);
    const int rk = __shfl_sync(0xffffffffu, rank, src);
    const bool hit = ((z >> lane) & 1u) && (__popc(z & ((1u << lane) - 1u)) == rk);
    const int bit = __ffs(__ballot_sync(0xffffffffu, hit)) - 1;
    if (lane == src) {
#pragma unroll
        for (int k = 0; k < NW; ++k)
            if (k == kk) w[k] |= 1u << bit;
        zl -= 1;
    }
    if (lane >= src) incl -= 1;
}

template <int NW>
__device__ __forceinline__ void lane_zero_scan(const uint32_t (&w)[NW], int lane, int& zl, int& incl, int& total) {
    zl = 0;
#pragma unroll
    for (int k = 0; k < NW; ++k) zl += __popc(~w[k]);
    incl = zl;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int t = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += t;
    }
    total = __shfl_sync(0xffffffffu, incl, 31);
}

// position of the n-th (0-based) set bit of m (which has more than n set bits): 5 popc steps, branch free
// (__fns compiles to a much longer sequence)
__device__ __forceinline__ int nth_set_bit(uint32_t m, int n) {
    int pos = 0;
#pragma unroll
    for (int w = 16; w >= 1; w >>= 1) {
        const int c = __popc(m & ((1u << w) - 1u));
        const bool up = n >= c;
        pos += up ? w : 0;
        n -= up ? c : 0;
        m = up ? (m >> w) : m;
    }
    return pos;
}

// q-th zero bit of a state stored as a plain word array (single thread).
__device__ __forceinline__ int kth_zero_serial(const uint32_t* s, int n_words, int q) {
    for (int k = 0; k < n_words; ++k) {
        const uint32_t z = ~s[k];
        const int pz = __popc(z);
        if (q < pz) return k * 32 + (int)__fns(z, 0, q + 1);
        q -= pz;
    }
    return -1;
}

// Grid-wide barrier on a monotonically increasing counter (zeroed by the host before the launch).
__device__ __forceinline__ void grid_barrier(unsigned* counter, unsigned& target) {
    __syncthreads();
    if (threadIdx.x == 0) {
        target += gridDim.x;
        __threadfence();                                   // publish this CTA's writes
        atomicAdd(counter, 1u);
        unsigned v;
        do {
            asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(counter) : "memory");
            if (v < target) __nanosleep(32);
        } while (v < target);
    }
    __syncthreads();
}

struct MctsArgs {
    const float *p, *size, *cost;
    const int32_t* guard;   // [A] guard (kill action) index per action, or nullptr
    const int32_t* cover;   // [A] cover (restore action) index per action, or nullptr (then no cover region in smem)
    int A;
    const uint32_t* root_state;
    int R, D, T;
    uint32_t k0, k1;
    float c, lo, inv_range;
    const float* lnN;
    int32_t* root_n;
    float* root_w;
    int32_t* num_nodes_out;
    // per-CTA tree replicas: replica b starts at base + b * stride (elements)
    int32_t* visits;     // [grid][T+1]
    int32_t* child_n;    // [grid][(T+1) * A_pad]
    float* child_w;
    int32_t* child_id;
    size_t node_stride;  // (T+1) rounded up to 64
    float* val;          // [2][R]  (double buffered across iterations)
    unsigned* barrier;   // grid barrier counter (zero at launch)
};

template <int NW>
__global__ void __launch_bounds__(MCTS_THREADS) mcts_search_kernel(MctsArgs P) {
    constexpr int A_PAD = 1024 * NW, NWORDS = 32 * NW;
    unsigned bar_target = 0;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    TermsS terms = carve_terms<NW>(smem_raw, smem_raw + mcts_smem_bytes<NW>());
    uint32_t* const s_scratch = reinterpret_cast<uint32_t*>(smem_raw + terms_smem_bytes<NW>()) + (threadIdx.x >> 5) * NWORDS;
    __shared__ uint32_t s_state[NWORDS];
    __shared__ int2 s_path[MAXD];
    __shared__ float s_key[MCTS_WARPS];
    __shared__ float s_tree[MCTS_WARPS];
    __shared__ int s_arg[MCTS_WARPS];
    __shared__ int s_node, s_depth, s_plen, s_created, s_stop, s_L0, s_numnodes;
    __shared__ int s_pref[NWORDS];                     // legal actions of the leaf state in the words before word k

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    // this CTA's replica of the tree (identical in every CTA: all apply the same deterministic updates)
    int32_t* const visits = P.visits + (size_t)blockIdx.x * P.node_stride;
    int32_t* const child_n = P.child_n + (size_t)blockIdx.x * P.node_stride * A_PAD;
    float* const child_w = P.child_w + (size_t)blockIdx.x * P.node_stride * A_PAD;
    int32_t* const child_id = P.child_id + (size_t)blockIdx.x * P.node_stride * A_PAD;
    stage_terms<NW>(P.p, P.size, P.cost, P.guard, P.cover, P.A, terms);
    // the replica is initialised here, by its own CTA (no host memsets): T+1 node rows
    for (size_t i = tid; i < (size_t)(P.T + 1) * A_PAD; i += MCTS_THREADS) { child_n[i] = 0; child_w[i] = 0.f; child_id[i] = -1; }
    for (int i = tid; i <= P.T; i += MCTS_THREADS) visits[i] = 0;
    if (tid == 0) s_numnodes = 1;                                        // the root
    __syncthreads();

    long long prof[4] = {0, 0, 0, 0}, tc0 = 0;
    const bool prof_on = blockIdx.x == 0 && tid == 0;
    for (int t = 0; t < P.T; ++t) {
        float* const val = P.val + (size_t)(t & 1) * P.R;
        if (prof_on) tc0 = clock64();
        // ------------------------------------------------------------------ select (redundant per CTA)
        for (int k = tid; k < NWORDS; k += MCTS_THREADS) {
            uint32_t wv = P.root_state ? P.root_state[k] : 0u;
            // padding bits (a >= A) are always applied
            const int a0 = k * 32;
            if (a0 + 32 > P.A) wv |= (a0 >= P.A) ? 0xffffffffu : (0xffffffffu << (P.A - a0));
            s_state[k] = wv;
        }
        // the legal count shrinks by one per level: L(depth) = L(root) - depth, L(root) computed once per iteration
        if (warp == 0) {
            __syncwarp();
            int z = 0;
            for (int k = lane; k < NWORDS; k += 32) {
                uint32_t wv = P.root_state ? P.root_state[k] : 0u;
                const int a0 = k * 32;
                if (a0 + 32 > P.A) wv |= (a0 >= P.A) ? 0xffffffffu : (0xffffffffu << (P.A - a0));
                z += __popc(~wv);
            }
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) z += __shfl_xor_sync(0xffffffffu, z, o);
            if (lane == 0) {
                s_node = 0; s_depth = 0; s_plen = 0; s_created = 0;
                s_L0 = z;                                                // legal actions at the root
                s_stop = (visits[0] == 0 || P.D <= 0 || z == 0) ? 1 : 0;
            }
        }
        __syncthreads();
        while (!s_stop) {                                                // s_stop is rewritten only between the two barriers below
            const int node = s_node;
            const float lnN = __ldg(P.lnN + visits[node]);
            float best_key = -INFINITY;
            int best_a = 0x7fffffff;
            const size_t base = (size_t)node * A_PAD;
            for (int a0 = tid; a0 < A_PAD; a0 += 2 * MCTS_THREADS) {     // two actions per pass: their loads travel together
                const int a1 = a0 + MCTS_THREADS;
                const bool ok0 = !((s_state[a0 >> 5] >> (a0 & 31)) & 1u);
                const bool ok1 = a1 < A_PAD && !((s_state[(a1 & (A_PAD - 1)) >> 5] >> (a1 & 31)) & 1u);
                const int n0 = ok0 ? child_n[base + a0] : 0, n1 = ok1 ? child_n[base + a1] : 0;
                const float cw0 = ok0 ? child_w[base + a0] : 0.f, cw1 = ok1 ? child_w[base + a1] : 0.f;
#pragma unroll
                for (int u = 0; u < 2; ++u) {                             // ascending a: strict > keeps the lowest
                    const bool ok = u ? ok1 : ok0;
                    const int n = u ? n1 : n0, a = u ? a1 : a0;
                    if (!ok) continue;
                    float key;
                    if (n == 0) {
                        key = INFINITY;
                    } else {
                        const float nf = (float)n;
                        const float q = __fdiv_rn(u ? cw1 : cw0, nf);
                        key = __fadd_rn(q, __fmul_rn(P.c, __fsqrt_rn(__fdiv_rn(lnN, nf))));
                    }
                    if (key > best_key) { best_key = key; best_a = a; }
                }
            }
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) {
                const float ok = __shfl_xor_sync(0xffffffffu, best_key, o);
                const int oa = __shfl_xor_sync(0xffffffffu, best_a, o);
                if (ok > best_key || (ok == best_key && oa < best_a)) { best_key = ok; best_a = oa; }
            }
            if (lane == 0) { s_key[warp] = best_key; s_arg[warp] = best_a; }
            __syncthreads();                                             // everyone has read s_stop / s_node / s_state
            if (warp == 0) {
                float bk = lane < MCTS_WARPS ? s_key[lane] : -INFINITY;
                int ba = lane < MCTS_WARPS ? s_arg[lane] : 0x7fffffff;
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) {
                    const float ok = __shfl_xor_sync(0xffffffffu, bk, o);
                    const int oa = __shfl_xor_sync(0xffffffffu, ba, o);
                    if (ok > bk || (ok == bk && oa < ba)) { bk = ok; ba = oa; }
                }
              if (lane == 0) {
                s_path[s_plen] = make_int2(node, ba);
                s_plen += 1;
                s_state[ba >> 5] |= 1u << (ba & 31);
                const int depth_new = s_depth + 1;
                s_depth = depth_new;
                const int cid = child_id[base + ba];
                if (cid < 0) {
                    s_created = 1; s_node = s_numnodes; s_stop = 1;      // new leaf
                } else {
                    s_node = cid;                                        // descend; stop at a terminal node
                    if (visits[cid] == 0 || depth_new >= P.D || s_L0 - depth_new == 0) s_stop = 1;
                }
              }
            }
            __syncthreads();
        }
        if (tid == 0) s_L0 = s_L0 - s_depth;                             // legal count of the leaf state
        if (warp == 1) {                                                 // exclusive prefix of the per-word legal counts (backup)
            int run = 0;
            for (int k0 = 0; k0 < NWORDS; k0 += 32) {
                const int z = __popc(~s_state[k0 + lane]);
                int inc = z;
#pragma unroll
                for (int o = 1; o < 32; o <<= 1) { const int t_ = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += t_; }
                s_pref[k0 + lane] = run + inc - z;
                run += __shfl_sync(0xffffffffu, inc, 31);
            }
        }
        __syncthreads();
        const int leaf = s_node, depth = s_depth, L0 = s_L0;
        const bool first_move = (P.D - depth) > 0 && L0 > 0;
        if (prof_on) { const long long c = clock64(); prof[0] += c - tc0; tc0 = c; }

        // ------------------------------------------------------------------ rollouts (warp per rollout)
        // (8 lanes per rollout / 4 rollouts per warp was tried: the per-step chain of dependent collectives got LONGER --
        // the n-th-set-bit search has to run inside one lane -- and with 7 instead of 28 warps per SM nothing hid it)
        // RANK-SPACE rollouts (round 2): a rollout applies "the j_k-th still-legal action" left times.  Instead of updating
        // the warp-distributed bitset at every step (ballot -> ffs -> 2 shfl -> popc -> ballot -> ffs: a chain of dependent
        // collectives, ~35 instructions), the picks are kept as a SORTED list of ranks among the leaf's legal actions, one
        // slot per lane (two registers: 64 slots): with s_0 < s_1 < ... the earlier picks and t_i = s_i - i (non-decreasing),
        // the j-th still-legal action has leaf rank j + c, c = #{i : t_i <= j} -- ONE ballot + popc -- and is inserted at
        // slot c (one shfl_up; the shifted entries lose 1).  The ranks become bit positions once, at the end (each lane
        // resolves its own picks: binary search over the per-word prefix counts + fns), scattered into a per-warp scratch
        // bitset.  Same draws, same set, hence the same state and -- same summation order -- the same reward, bit for bit.
        const bool rank_path = (P.D - depth) <= 64;
        for (int r = (int)blockIdx.x * MCTS_WARPS + warp; rank_path && r < P.R; r += (int)gridDim.x * MCTS_WARPS) {
            int left = P.D - depth;
            int L = L0, n = 0;
            int t_lo = 0x7fffffff, t_hi = 0x7fffffff;                    // slot lane / lane + 32; empty = +inf
            auto pick = [&](int j) {
                if (n < 32) {                                             // (uniform) the upper half is still empty
                    const int c = __popc(__ballot_sync(0xffffffffu, t_lo <= j));
                    const int up = __shfl_up_sync(0xffffffffu, t_lo, 1);
                    t_lo = (lane < c) ? t_lo : (lane == c ? j : up - 1);
                } else {
                    const int c = __popc(__ballot_sync(0xffffffffu, t_lo <= j)) + __popc(__ballot_sync(0xffffffffu, t_hi <= j));
                    const int up_lo = __shfl_up_sync(0xffffffffu, t_lo, 1);
                    int up_hi = __shfl_up_sync(0xffffffffu, t_hi, 1);
                    const int carry = __shfl_sync(0xffffffffu, t_lo, 31);
                    if (lane == 0) up_hi = carry;
                    t_lo = (lane < c) ? t_lo : (lane == c ? j : up_lo - 1);
                    t_hi = (lane + 32 < c) ? t_hi : (lane + 32 == c ? j : up_hi - 1);
                }
                ++n;
            };
            if (first_move) { pick(r % L0); L -= 1; left -= 1; }
            // every Philox block of the rollout at once: lane i computes block i (counter (r, i, t, 0)) -- at most 16 blocks
            // for <= 64 steps -- instead of all 32 lanes computing the same block 13 times over (~100 instructions each)
            uint32_t rnd[4];
            philox4x32_10((uint32_t)r, (uint32_t)lane, (uint32_t)t, 0u, P.k0, P.k1, rnd);
            const int nsteps = left < L ? left : L;                      // a step removes one legal action: min(left, L) steps
            for (int k = 0; k < nsteps; k += 4) {                         // one Philox block feeds four steps
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                    const uint32_t x = __shfl_sync(0xffffffffu, rnd[q], k >> 2);
                    if (k + q < nsteps) pick((int)__umulhi(x, (uint32_t)(L - (k + q))));
                }
            }
            // ranks -> bits: scratch = leaf state, then every pick sets its bit
#pragma unroll
            for (int k = 0; k < NW; ++k) s_scratch[lane * NW + k] = s_state[lane * NW + k];
            __syncwarp();
#pragma unroll
            for (int half = 0; half < 2; ++half) {
                const int slot = lane + 32 * half;
                if (slot < n) {
                    const int q = (half ? t_hi : t_lo) + slot;           // rank among the leaf's legal actions
                    int lo_w = 0, hi_w = NWORDS - 1;                     // last word whose prefix count is <= q
                    while (lo_w < hi_w) {
                        const int mid = (lo_w + hi_w + 1) >> 1;
                        if (s_pref[mid] <= q) lo_w = mid; else hi_w = mid - 1;
                    }
                    const int bit = nth_set_bit(~s_state[lo_w], q - s_pref[lo_w]);
                    atomicOr(&s_scratch[lo_w], 1u << bit);
                }
            }
            __syncwarp();
            uint32_t w[NW];
#pragma unroll
            for (int k = 0; k < NW; ++k) w[k] = s_scratch[lane * NW + k];
            __syncwarp();                                                 // the scratch is reused by this warp's next rollout
            const float sc = warp_score<NW>(w, terms, lane);
            if (lane == 0) val[r] = __fmul_rn(__fsub_rn(sc, P.lo), P.inv_range);
        }
        // deeper rollouts (more than 64 steps below the leaf): the per-step bitset update
        for (int r = (int)blockIdx.x * MCTS_WARPS + warp; !rank_path && r < P.R; r += (int)gridDim.x * MCTS_WARPS) {
            uint32_t w[NW];
#pragma unroll
            for (int k = 0; k < NW; ++k) w[k] = s_state[lane * NW + k];
            int left = P.D - depth;
            int zl, incl, L;
            lane_zero_scan<NW>(w, lane, zl, incl, L);                     // once; maintained incrementally below
            if (first_move) {
                apply_jth<NW>(w, zl, incl, r % L0, lane);
                L -= 1; left -= 1;
            }
            for (int k = 0; k < left && L > 0; k += 4) {                  // one Philox call feeds four steps
                uint32_t rnd[4];
                philox4x32_10((uint32_t)r, (uint32_t)(k >> 2), (uint32_t)t, 0u, P.k0, P.k1, rnd);
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                    if (k + q < left && L > 0) {
                        const int j = (int)__umulhi(rnd[q], (uint32_t)L);
                        apply_jth<NW>(w, zl, incl, j, lane);
                        L -= 1;
                    }
                }
            }
            const float sc = warp_score<NW>(w, terms, lane);
            if (lane == 0) val[r] = __fmul_rn(__fsub_rn(sc, P.lo), P.inv_range);
        }
        if (prof_on) { const long long c = clock64(); prof[1] += c - tc0; tc0 = c; }
        grid_barrier(P.barrier, bar_target);                             // every rollout value of this iteration is visible
        if (prof_on) { const long long c = clock64(); prof[2] += c - tc0; tc0 = c; }

        // ------------------------------------------------------------------ backup (every CTA, on its own replica)
        // the tree-sum operands are requested first, so their L2 latency overlaps the leaf-children pass
        constexpr int TS = 512;                                         // threads used by the tree sum (power of two)
        const int m = P.R >= TS ? P.R / TS : 1;
        const int nthr = P.R / m;                                       // power of two <= TS
        float loc[MAXR / TS];
        if (tid < nthr)
            for (int i = 0; i < m; ++i) loc[i] = __ldcg(val + tid * m + i);
        if (first_move) {   // leaf children: action a has rank q among the leaf's legal actions; fixed ascending-r accumulation
            const int nq = P.R < L0 ? P.R : L0;
            const size_t lbase = (size_t)leaf * A_PAD;
            // the leaf was created THIS iteration or is terminal-by-depth: in both cases its child row is read here for the
            // first time in this iteration, and a new leaf's row is still all zero -- so the row's old values are only loaded
            // when the leaf already existed
            const bool fresh = s_created != 0;
            for (int a0 = tid; a0 < A_PAD; a0 += 2 * MCTS_THREADS) {     // two actions per pass: one latency round for both
                int aa[2], qq[2];
                bool on[2];
                float wsum[2];
                int cnt[2];
#pragma unroll
                for (int u = 0; u < 2; ++u) {
                    const int a = a0 + u * MCTS_THREADS;
                    aa[u] = a;
                    const uint32_t wv = s_state[(a & (A_PAD - 1)) >> 5];
                    qq[u] = __popc(~wv & ((1u << (a & 31)) - 1u)) + s_pref[(a & (A_PAD - 1)) >> 5];   // legal actions below a
                    on[u] = a < A_PAD && !((wv >> (a & 31)) & 1u) && qq[u] < nq;                      // legal at the leaf, has rollouts
                    wsum[u] = (on[u] && !fresh) ? child_w[lbase + a] : 0.f;
                    cnt[u] = (on[u] && !fresh) ? child_n[lbase + a] : 0;
                }
                float v[2][4];
                int r[2] = {qq[0], qq[1]};
                bool more = true;
                while (more) {                                            // four loads per action in flight, added in ascending r
                    more = false;
#pragma unroll
                    for (int u = 0; u < 2; ++u)
#pragma unroll
                        for (int i = 0; i < 4; ++i)
                            if (on[u] && r[u] + i * L0 < P.R) v[u][i] = __ldcg(val + r[u] + i * L0);
#pragma unroll
                    for (int u = 0; u < 2; ++u) {
#pragma unroll
                        for (int i = 0; i < 4; ++i)
                            if (on[u] && r[u] + i * L0 < P.R) { wsum[u] = __fadd_rn(wsum[u], v[u][i]); ++cnt[u]; }
                        r[u] += 4 * L0;
                        more = more || (on[u] && r[u] < P.R);
                    }
                }
#pragma unroll
                for (int u = 0; u < 2; ++u)
                    if (on[u]) { child_w[lbase + aa[u]] = wsum[u]; child_n[lbase + aa[u]] = cnt[u]; }
            }
        }
        {
            // adjacent-pairs tree sum of val[0..R): each thread reduces an aligned block of m values in
            // registers / local memory, lanes combine with the xor butterfly (== adjacent pairs, lane i holds
            // block i), warps with a fixed pairing.  Same tree as the oracle for any power-of-two R.
            float v = 0.f;
            if (tid < nthr) {
                for (int st = 1; st < m; st <<= 1)
                    for (int i = 0; i < m; i += 2 * st) loc[i] = __fadd_rn(loc[i], loc[i + st]);
                v = loc[0];
            }
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const float other = __shfl_xor_sync(0xffffffffu, v, o);
                if (o < nthr) v = __fadd_rn(v, other);
            }
            if (lane == 0) s_tree[warp] = v;
            __syncthreads();
            float total = s_tree[0];
            if (nthr > 32) {                                            // second level: warp sums, same adjacent pairing
                const int nw = nthr / 32;                               // 2, 4, 8 or 16
                float u = (warp == 0 && lane < nw) ? s_tree[lane] : 0.f;
#pragma unroll
                for (int o = 1; o < 16; o <<= 1) {
                    const float other = __shfl_xor_sync(0xffffffffu, u, o);
                    if (o < nw) u = __fadd_rn(u, other);
                }
                __syncthreads();                                        // every thread has read s_tree[0] above
                if (tid == 0) s_tree[0] = u;
                __syncthreads();
                total = s_tree[0];
            }
            const int plen = s_plen;
            for (int i = tid; i < plen; i += MCTS_THREADS) {
                const int2 e = s_path[i];
                const size_t idx = (size_t)e.x * A_PAD + e.y;
                child_n[idx] = child_n[idx] + P.R;
                child_w[idx] = __fadd_rn(child_w[idx], total);
                visits[e.x] = visits[e.x] + 1;
            }
            if (tid == 0) {
                visits[leaf] = visits[leaf] + 1;
                if (s_created) {
                    const int2 e = s_path[plen - 1];
                    child_id[(size_t)e.x * A_PAD + e.y] = leaf;
                    s_numnodes = s_numnodes + 1;
                }
            }
        }
        __syncthreads();                                                 // this CTA's replica is up to date for its next select
        if (prof_on) { const long long c = clock64(); prof[3] += c - tc0; tc0 = c; }
    }
    if (prof_on) {                                                       // phase cycle counts of CTA 0 (diagnostics; 4 words after the barrier counter)
        for (int i = 0; i < 4; ++i) P.barrier[8 + i] = (unsigned)(prof[i] >> 4);
    }
    // ---------------------------------------------------------------------- outputs
    if (blockIdx.x == 0) {
        for (int a = tid; a < A_PAD; a += MCTS_THREADS) {
            P.root_n[a] = child_n[a];
            P.root_w[a] = child_w[a];
        }
        if (tid == 0) *P.num_nodes_out = s_numnodes;
    }
}

// ------------------------------------------------------------------------------------------ rewards.score
template <int NW>
__global__ void __launch_bounds__(256) reward_score_kernel(const uint32_t* __restrict__ states, int64_t B,
                                                           const float* __restrict__ p, const float* __restrict__ size,
                                                           const float* __restrict__ cost, const int32_t* __restrict__ guard,
                                                           const int32_t* __restrict__ cover, int A, float* __restrict__ out) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    TermsS terms = carve_terms<NW>(smem_raw, smem_raw + terms_smem_bytes<NW>());
    stage_terms<NW>(p, size, cost, guard, cover, A, terms);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int64_t s = (int64_t)blockIdx.x * 8 + warp; s < B; s += (int64_t)gridDim.x * 8) {
        uint32_t w[NW];
#pragma unroll
        for (int k = 0; k < NW; ++k) w[k] = states[s * (32 * NW) + lane * NW + k];
        const float sc = warp_score<NW>(w, terms, lane);
        if (lane == 0) out[s] = sc;
    }
}

// ------------------------------------------------------------------------------------------ plan(): validate and commit
// The commit loop of ai.planner.mcts.plan ("sandbox validates, then apply", architecture.mdx:81-86) on the device.  After a tree
// search the ranked root children are validated with the EXACT reward: repeatedly, every remaining candidate c is scored as
// score(state + c) (the spec'd fixed-order fp32 sum: warp_score), the highest-ranked candidate that improves on the current
// score is committed, and only candidates that still looked improving stay in the list -- up to max_commits times.  With
// thousands of candidates and 64 commits per search this loop was ~90 % of the planner's wall time when every round was a
// host round trip (states up, scores down).  Here: one cooperative launch, one grid barrier per round; every CTA keeps its
// own copy of the state and of the candidate list and applies the (deterministic) round result to it, the round's scores /
// flags travel through double-buffered global arrays.  Bit-identical decisions and scores to the host loop.
struct CommitArgs {
    const float *p, *size, *cost;
    const int32_t* guard;
    const int32_t* cover;       // nullptr, or [A] (then the cover region follows the candidate list in smem)
    int A;
    uint32_t* state;            // [32*NW] in: the current state, out: the state after the commits
    const int32_t* cand;        // [n_cand] ranked candidates
    int n_cand, max_commits, allow_tentative;
    float cur;                  // exact score of `state`
    float* sc_buf;              // [2][cap] scores of the round
    int32_t* flag_buf;          // [2][cap] 1 = improves
    int cap;
    int32_t* actions_out;       // [max_commits]
    float* scores_out;          // [max_commits]
    int32_t* n_out;             // [0] commits made, [1] candidates left that still looked improving
    unsigned* barrier;          // zero at launch
};

template <int NW>
__global__ void __launch_bounds__(256) plan_commit_kernel(CommitArgs P) {
    constexpr int NWORDS = 32 * NW;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    TermsS terms = carve_terms<NW>(smem_raw, smem_raw + terms_smem_bytes<NW>() + 4096 * 4);
    int32_t* s_cand = reinterpret_cast<int32_t*>(smem_raw + terms_smem_bytes<NW>());          // [cap]
    __shared__ uint32_t s_state[NWORDS];
    __shared__ int s_first, s_cnt[8];
    __shared__ float s_cur;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    unsigned bar_target = 0;
    stage_terms<NW>(P.p, P.size, P.cost, P.guard, P.cover, P.A, terms);
    for (int i = tid; i < P.n_cand; i += 256) s_cand[i] = P.cand[i];
    for (int k = tid; k < NWORDS; k += 256) s_state[k] = P.state[k];
    if (tid == 0) s_cur = P.cur;
    __syncthreads();
    int n = P.n_cand, committed = 0;
    const int gw = (int)blockIdx.x * 8 + warp, GW = (int)gridDim.x * 8;
    for (int round = 0; n > 0 && committed < P.max_commits; ++round) {
        float* sc = P.sc_buf + (size_t)(round & 1) * P.cap;
        int32_t* fl = P.flag_buf + (size_t)(round & 1) * P.cap;
        const float cur = s_cur;
        for (int i = gw; i < n; i += GW) {                                // score(state + candidate i): one warp each
            const int a = s_cand[i];
            uint32_t w[NW];
#pragma unroll
            for (int k = 0; k < NW; ++k) {
                w[k] = s_state[lane * NW + k];
                if ((a >> 5) == lane * NW + k) w[k] |= 1u << (a & 31);
            }
            const float v = warp_score<NW>(w, terms, lane);
            if (lane == 0) { sc[i] = v; fl[i] = v > cur ? 1 : 0; }
        }
        grid_barrier(P.barrier, bar_target);                              // the round's scores are visible to every CTA
        // every CTA, redundantly: the first improving candidate; the improving candidates after it form the next list
        if (tid == 0) s_first = 0x7fffffff;
        __syncthreads();
        int my_first = 0x7fffffff;
        for (int i = tid; i < n; i += 256)
            if (__ldcg(fl + i)) { my_first = i; break; }
        if (my_first != 0x7fffffff) atomicMin(&s_first, my_first);
        __syncthreads();
        int first = s_first;
        bool tentative = false;
        if (first == 0x7fffffff) {
            if (P.allow_tentative && committed == 0) { first = 0; tentative = true; }   // lookahead: the search's recommendation
            else break;                                                   // (uniform: every thread read the same s_first)
        }
        // stable compaction of {i > first : fl[i]} into the front of s_cand (blocked: thread t owns a contiguous chunk)
        const int chunk = (n + 255) / 256;
        const int lo = tid * chunk, hi = min(lo + chunk, n);
        int cnt = 0;
        if (!tentative)
            for (int i = max(lo, first + 1); i < hi; ++i) cnt += __ldcg(fl + i);
        int inc = cnt;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const int t_ = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += t_; }
        if (lane == 31) s_cnt[warp] = inc;
        const int a_first = s_cand[first];
        const float new_cur = __ldcg(sc + first);
        __syncthreads();                                                  // s_cnt complete; every thread has read s_cand[first]
        int base = inc - cnt;
        for (int w_ = 0; w_ < warp; ++w_) base += s_cnt[w_];
        int total = 0;
        for (int w_ = 0; w_ < 8; ++w_) total += s_cnt[w_];
        int keep[16];                                                     // chunk <= 16 for cap <= 4096
        int nk = 0;
        if (!tentative)
            for (int i = max(lo, first + 1); i < hi; ++i)
                if (__ldcg(fl + i)) keep[nk++] = s_cand[i];
        __syncthreads();                                                  // all reads of the old list are done
        for (int j = 0; j < nk; ++j) s_cand[base + j] = keep[j];
        if (tid == 0) {
            s_state[a_first >> 5] |= 1u << (a_first & 31);
            s_cur = new_cur;
            if (blockIdx.x == 0) { P.actions_out[committed] = a_first; P.scores_out[committed] = new_cur; }
        }
        __syncthreads();
        n = total;
        committed += 1;
    }
    if (blockIdx.x == 0) {
        for (int k = tid; k < NWORDS; k += 256) P.state[k] = s_state[k];
        if (tid == 0) { P.n_out[0] = committed; P.n_out[1] = n; }
    }
}

static int nw_for(int A) { return A <= 1024 ? 1 : (A <= 2048 ? 2 : 4); }

static int mcts_grid_for(int R) {
    int want = (R + MCTS_WARPS - 1) / MCTS_WARPS;
    if (want < 1) want = 1;
    const int sms = sm_count();
    return want < sms ? want : sms;                // one CTA per SM (896 threads + the staged terms fill an SM)
}

struct MctsLayout {
    size_t visits, child_n, child_w, child_id, val, barrier, total, node_stride;
    int grid;
};
static MctsLayout mcts_layout(int A, int T, int R) {
    const size_t A_pad = 1024 * (size_t)nw_for(A);
    auto al = [](size_t v) { return (v + 255) & ~(size_t)255; };
    MctsLayout L;
    L.grid = mcts_grid_for(R);
    L.node_stride = ((size_t)T + 1 + 63) & ~(size_t)63;
    const size_t per_tree = L.node_stride * A_pad * 4;
    size_t o = 0;
    L.barrier = o; o = al(o + 4);
    L.visits = o; o = al(o + (size_t)L.grid * L.node_stride * 4);
    L.child_n = o; o = al(o + (size_t)L.grid * per_tree);
    L.child_w = o; o = al(o + (size_t)L.grid * per_tree);
    L.child_id = o; o = al(o + (size_t)L.grid * per_tree);
    L.val = o; o = al(o + (size_t)2 * R * 4);
    L.total = o;
    return L;
}

template <int NW>
static int launch_mcts(MctsArgs& args, int grid, cudaStream_t st) {
    const size_t smem = mcts_smem_bytes<NW>() + (args.cover ? cover_smem_bytes<NW>() : 0);
    const int rc = set_max_dynamic_smem((const void*)mcts_search_kernel<NW>, smem);
    if (rc) return rc;
    int per_sm = 0;
    NERRF_CHECK_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, mcts_search_kernel<NW>, MCTS_THREADS, smem));
    NERRF_REQUIRE(per_sm >= 1, "mcts kernel does not fit on an SM");
    void* kargs[] = {(void*)&args};
    NERRF_CHECK_CUDA(cudaLaunchCooperativeKernel((void*)mcts_search_kernel<NW>, dim3(grid), dim3(MCTS_THREADS), kargs, smem, st));
    return NERRF_OK;
}

}  // namespace nerrf

using namespace nerrf;

// Spec v2 cover table check (host side; `cover` / `guard` may be host or device pointers).  cover[a] is -1 or the index
// of a restore action in word 0 (< 32, < A), never a itself; a restore action is not covered itself (one level), and no
// index is both a guard and a cover target.
static int check_cover(const int32_t* cover, const int32_t* guard, int A, cudaStream_t st) {
    if (!cover) return NERRF_OK;
    std::vector<int32_t> c((size_t)A), g((size_t)A, -1);
    NERRF_CHECK_CUDA(cudaMemcpyAsync(c.data(), cover, (size_t)A * 4, cudaMemcpyDefault, st));
    if (guard) NERRF_CHECK_CUDA(cudaMemcpyAsync(g.data(), guard, (size_t)A * 4, cudaMemcpyDefault, st));
    NERRF_CHECK_CUDA(cudaStreamSynchronize(st));
    const int lim = A < 32 ? A : 32;
    bool target[32] = {false}, guard_target[32] = {false};
    for (int a = 0; a < A; ++a) {
        NERRF_REQUIRE(c[a] == -1 || (c[a] >= 0 && c[a] < lim), "cover[%d] = %d: must be -1 or a restore action index in 0..%d",
                      a, c[a], lim - 1);
        NERRF_REQUIRE(c[a] != a, "cover[%d] names the action itself", a);
        if (c[a] >= 0) target[c[a]] = true;
        if (g[a] >= 0 && g[a] < 32) guard_target[g[a]] = true;
    }
    for (int r = 0; r < lim; ++r) {
        NERRF_REQUIRE(!target[r] || c[r] == -1, "restore action %d is itself covered (covers do not chain)", r);
        NERRF_REQUIRE(!(target[r] && guard_target[r]), "action %d is both a guard and a cover target", r);
    }
    return NERRF_OK;
}

extern "C" int nerrf_reward_score_ex(const uint32_t* states, int64_t B, const float* p, const float* size,
                                     const float* cost, const int32_t* guard, const int32_t* cover, int A, float* out,
                                     nerrf_stream_t stream) {
    NERRF_REQUIRE(states && p && size && cost && out, "null pointer");
    NERRF_REQUIRE(A >= 1 && A <= 4096, "number of actions must be in 1..4096 (got %d)", A);
    NERRF_REQUIRE(B >= 0, "negative batch");
    cudaStream_t st = (cudaStream_t)stream;
    const int rc0 = check_cover(cover, guard, A, st);
    if (rc0) return rc0;
    if (B == 0) return NERRF_OK;
    const int NW = nw_for(A);
    int64_t g = (B + 7) / 8;
    const int64_t cap = (int64_t)sm_count() * 8;
    if (g > cap) g = cap;
    auto go = [&](auto kern, size_t smem) -> int {
        if (smem > 48 * 1024) {                                           // staged terms above the 48 KB default
            const int rc = set_max_dynamic_smem((const void*)kern, smem);
            if (rc) return rc;
        }
        kern<<<(unsigned)g, 256, smem, st>>>(states, B, p, size, cost, guard, cover, A, out);
        return launch_status("reward_score_kernel");
    };
    if (NW == 1) return go(reward_score_kernel<1>, terms_smem_bytes<1>() + (cover ? cover_smem_bytes<1>() : 0));
    if (NW == 2) return go(reward_score_kernel<2>, terms_smem_bytes<2>() + (cover ? cover_smem_bytes<2>() : 0));
    return go(reward_score_kernel<4>, terms_smem_bytes<4>() + (cover ? cover_smem_bytes<4>() : 0));
}

extern "C" int nerrf_reward_score(const uint32_t* states, int64_t B, const float* p, const float* size,
                                  const float* cost, const int32_t* guard, int A, float* out, nerrf_stream_t stream) {
    return nerrf_reward_score_ex(states, B, p, size, cost, guard, nullptr, A, out, stream);
}

extern "C" int nerrf_mcts_workspace_bytes(int A, int T, int R, size_t* bytes) {
    NERRF_REQUIRE(bytes, "null out");
    NERRF_REQUIRE(A >= 1 && A <= 4096, "number of actions must be in 1..4096 (got %d)", A);
    NERRF_REQUIRE(T >= 1 && T <= (1 << 20), "iterations out of range");
    NERRF_REQUIRE(R >= 1 && R <= MAXR && (R & (R - 1)) == 0, "R must be a power of two in 1..%d (got %d)", MAXR, R);
    *bytes = mcts_layout(A, T, R).total;
    return NERRF_OK;
}

extern "C" int nerrf_mcts_search_ex(const float* p, const float* size, const float* cost, const int32_t* guard,
                                    const int32_t* cover, int A, const uint32_t* root_state, int R, int D, int T, uint64_t seed,
                                    float c, float lo, float inv_range, const float* ln_table, int32_t* root_n, float* root_w,
                                    int32_t* num_nodes, void* workspace, size_t workspace_bytes, nerrf_stream_t stream) {
    size_t need = 0;
    int rc = nerrf_mcts_workspace_bytes(A, T, R, &need);
    if (rc) return rc;
    NERRF_REQUIRE(p && size && cost && ln_table && root_n && root_w && num_nodes && workspace, "null pointer");
    NERRF_REQUIRE(D >= 0 && D <= MAXD, "depth must be in 0..%d (got %d)", MAXD, D);
    if (workspace_bytes < need) {
        set_error("mcts workspace too small: need %zu bytes, got %zu", need, workspace_bytes);
        return NERRF_ERR_WORKSPACE;
    }
    cudaStream_t st = (cudaStream_t)stream;
    rc = check_cover(cover, guard, A, st);
    if (rc) return rc;
    const MctsLayout L = mcts_layout(A, T, R);
    unsigned char* ws = (unsigned char*)workspace;
    NERRF_CHECK_CUDA(cudaMemsetAsync(ws + L.barrier, 0, 4, st));       // the tree replicas are initialised by the kernel itself
    MctsArgs a;
    a.p = p; a.size = size; a.cost = cost; a.guard = guard; a.cover = cover; a.A = A; a.root_state = root_state; a.R = R; a.D = D; a.T = T;
    a.k0 = (uint32_t)(seed & 0xffffffffu); a.k1 = (uint32_t)(seed >> 32);
    a.c = c; a.lo = lo; a.inv_range = inv_range; a.lnN = ln_table;
    a.root_n = root_n; a.root_w = root_w; a.num_nodes_out = num_nodes;
    a.visits = (int32_t*)(ws + L.visits); a.child_n = (int32_t*)(ws + L.child_n); a.child_w = (float*)(ws + L.child_w);
    a.child_id = (int32_t*)(ws + L.child_id); a.node_stride = L.node_stride; a.val = (float*)(ws + L.val);
    a.barrier = (unsigned*)(ws + L.barrier);
    const int NW = nw_for(A);
    if (NW == 1) return launch_mcts<1>(a, L.grid, st);
    if (NW == 2) return launch_mcts<2>(a, L.grid, st);
    return launch_mcts<4>(a, L.grid, st);
}

extern "C" int nerrf_mcts_search(const float* p, const float* size, const float* cost, const int32_t* guard, int A,
                                 const uint32_t* root_state, int R, int D, int T, uint64_t seed, float c, float lo,
                                 float inv_range, const float* ln_table, int32_t* root_n, float* root_w, int32_t* num_nodes,
                                 void* workspace, size_t workspace_bytes, nerrf_stream_t stream) {
    return nerrf_mcts_search_ex(p, size, cost, guard, nullptr, A, root_state, R, D, T, seed, c, lo, inv_range, ln_table, root_n,
                                root_w, num_nodes, workspace, workspace_bytes, stream);
}

// ---- host-buffer session: device memory + a stream live in the handle, so a host-side search is copies + one launch
struct nerrf_mcts_session {
    unsigned char* d = nullptr;
    size_t bytes = 0;
    int A_max = 0, T_max = 0, R_max = 0;
    cudaStream_t st = nullptr;
    size_t o_p, o_s, o_c, o_g, o_cv, o_rs, o_ln, o_rn, o_rw, o_nn, o_ws, ws_bytes;
};

extern "C" int nerrf_mcts_session_create(int A_max, int T_max, int R_max, nerrf_mcts_session** out) {
    NERRF_REQUIRE(out, "null out");
    size_t need = 0;
    int rc = nerrf_mcts_workspace_bytes(A_max, T_max, R_max, &need);
    if (rc) return rc;
    nerrf_mcts_session* s = new nerrf_mcts_session();
    s->A_max = A_max; s->T_max = T_max; s->R_max = R_max;
    const size_t A_pad = 1024 * (size_t)nw_for(A_max), nwords = 32 * (size_t)nw_for(A_max);
    auto al = [](size_t v) { return (v + 255) & ~(size_t)255; };
    s->o_p = 0; s->o_s = al(s->o_p + A_pad * 4); s->o_c = al(s->o_s + A_pad * 4); s->o_g = al(s->o_c + A_pad * 4);
    s->o_cv = al(s->o_g + A_pad * 4); s->o_rs = al(s->o_cv + A_pad * 4); s->o_ln = al(s->o_rs + nwords * 4); s->o_rn = al(s->o_ln + (size_t)(T_max + 2) * 4);
    s->o_rw = al(s->o_rn + A_pad * 4); s->o_nn = al(s->o_rw + A_pad * 4); s->o_ws = al(s->o_nn + 4);
    s->ws_bytes = need; s->bytes = s->o_ws + need;
    cudaError_t e = cudaMalloc((void**)&s->d, s->bytes);
    if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&s->st, cudaStreamNonBlocking);
    if (e != cudaSuccess) {
        set_error("mcts session: %s", cudaGetErrorString(e));
        if (s->d) cudaFree(s->d);
        delete s;
        return NERRF_ERR_CUDA;
    }
    *out = s;
    return NERRF_OK;
}

extern "C" int nerrf_mcts_session_destroy(nerrf_mcts_session* s) {
    if (!s) return NERRF_OK;
    if (s->st) cudaStreamDestroy(s->st);
    if (s->d) cudaFree(s->d);
    delete s;
    return NERRF_OK;
}

extern "C" int nerrf_mcts_session_search_host_ex(nerrf_mcts_session* s, const float* p, const float* size, const float* cost,
                                                 const int32_t* guard, const int32_t* cover, int A,
                                                 const uint32_t* root_state_host, int R, int D, int T, uint64_t seed, float c,
                                                 float lo, float inv_range, const float* ln_table_host, int32_t* root_n_host,
                                                 float* root_w_host, int32_t* num_nodes_host) {
    NERRF_REQUIRE(s && p && size && cost && ln_table_host && root_n_host && root_w_host && num_nodes_host, "null pointer");
    NERRF_REQUIRE(A >= 1 && A <= s->A_max && nw_for(A) == nw_for(s->A_max) && T >= 1 && T <= s->T_max && R >= 1 && R <= s->R_max,
                  "search (A=%d, T=%d, R=%d) exceeds the session (A_max=%d with the same word count, T_max=%d, R_max=%d)", A, T, R,
                  s->A_max, s->T_max, s->R_max);
    const size_t A_pad = 1024 * (size_t)nw_for(A), nwords = 32 * (size_t)nw_for(A);
    unsigned char* d = s->d;
    cudaStream_t st = s->st;
    NERRF_CHECK_CUDA(cudaMemcpyAsync(d + s->o_p, p, (size_t)A * 4, cudaMemcpyHostToDevice, st));
    NERRF_CHECK_CUDA(cudaMemcpyAsync(d + s->o_s, size, (size_t)A * 4, cudaMemcpyHostToDevice, st));
    NERRF_CHECK_CUDA(cudaMemcpyAsync(d + s->o_c, cost, (size_t)A * 4, cudaMemcpyHostToDevice, st));
    if (guard) NERRF_CHECK_CUDA(cudaMemcpyAsync(d + s->o_g, guard, (size_t)A * 4, cudaMemcpyHostToDevice, st));
    if (cover) NERRF_CHECK_CUDA(cudaMemcpyAsync(d + s->o_cv, cover, (size_t)A * 4, cudaMemcpyHostToDevice, st));
    if (root_state_host) NERRF_CHECK_CUDA(cudaMemcpyAsync(d + s->o_rs, root_state_host, nwords * 4, cudaMemcpyHostToDevice, st));
    NERRF_CHECK_CUDA(cudaMemcpyAsync(d + s->o_ln, ln_table_host, (size_t)(T + 2) * 4, cudaMemcpyHostToDevice, st));
    int rc = nerrf_mcts_search_ex((const float*)(d + s->o_p), (const float*)(d + s->o_s), (const float*)(d + s->o_c),
                               guard ? (const int32_t*)(d + s->o_g) : nullptr, cover ? (const int32_t*)(d + s->o_cv) : nullptr, A,
                               root_state_host ? (const uint32_t*)(d + s->o_rs) : nullptr, R, D, T, seed, c, lo, inv_range,
                               (const float*)(d + s->o_ln), (int32_t*)(d + s->o_rn), (float*)(d + s->o_rw), (int32_t*)(d + s->o_nn),
                               d + s->o_ws, s->ws_bytes, st);
    if (rc) return rc;
    NERRF_CHECK_CUDA(cudaMemcpyAsync(root_n_host, d + s->o_rn, A_pad * 4, cudaMemcpyDeviceToHost, st));
    NERRF_CHECK_CUDA(cudaMemcpyAsync(root_w_host, d + s->o_rw, A_pad * 4, cudaMemcpyDeviceToHost, st));
    NERRF_CHECK_CUDA(cudaMemcpyAsync(num_nodes_host, d + s->o_nn, 4, cudaMemcpyDeviceToHost, st));
    NERRF_CHECK_CUDA(cudaStreamSynchronize(st));
    return launch_status("mcts session search");
}

extern "C" int nerrf_mcts_session_search_host(nerrf_mcts_session* s, const float* p, const float* size, const float* cost,
                                              const int32_t* guard, int A, const uint32_t* root_state_host, int R, int D, int T,
                                              uint64_t seed, float c, float lo, float inv_range, const float* ln_table_host,
                                              int32_t* root_n_host, float* root_w_host, int32_t* num_nodes_host) {
    return nerrf_mcts_session_search_host_ex(s, p, size, cost, guard, nullptr, A, root_state_host, R, D, T, seed, c, lo, inv_range,
                                             ln_table_host, root_n_host, root_w_host, num_nodes_host);
}

// one-shot convenience: a temporary session (allocates and frees device memory inside the call)
extern "C" int nerrf_mcts_search_host_ex(const float* p, const float* size, const float* cost, const int32_t* guard,
                                         const int32_t* cover, int A, const uint32_t* root_state_host, int R, int D, int T,
                                         uint64_t seed, float c, float lo, float inv_range, const float* ln_table_host,
                                         int32_t* root_n_host, float* root_w_host, int32_t* num_nodes_host) {
    nerrf_mcts_session* s = nullptr;
    int rc = nerrf_mcts_session_create(A, T, R, &s);
    if (rc) return rc;
    rc = nerrf_mcts_session_search_host_ex(s, p, size, cost, guard, cover, A, root_state_host, R, D, T, seed, c, lo, inv_range,
                                           ln_table_host, root_n_host, root_w_host, num_nodes_host);
    nerrf_mcts_session_destroy(s);
    return rc;
}

extern "C" int nerrf_mcts_search_host(const float* p, const float* size, const float* cost, const int32_t* guard, int A,
                                      const uint32_t* root_state_host, int R, int D, int T, uint64_t seed, float c,
                                      float lo, float inv_range, const float* ln_table_host, int32_t* root_n_host,
                                      float* root_w_host, int32_t* num_nodes_host) {
    return nerrf_mcts_search_host_ex(p, size, cost, guard, nullptr, A, root_state_host, R, D, T, seed, c, lo, inv_range,
                                     ln_table_host, root_n_host, root_w_host, num_nodes_host);
}

extern "C" int nerrf_plan_commit_workspace_bytes(int n_cand_max, size_t* bytes) {
    NERRF_REQUIRE(bytes && n_cand_max >= 0 && n_cand_max <= 4096, "n_cand_max must be in 0..4096");
    *bytes = (size_t)4096 * 16 + 256;
    return NERRF_OK;
}

extern "C" int nerrf_plan_commit_ex(const float* p, const float* size, const float* cost, const int32_t* guard,
                                    const int32_t* cover, int A, uint32_t* state, const int32_t* cand, int n_cand, float cur,
                                    int max_commits, int allow_tentative, int32_t* actions_out, float* scores_out, int32_t* n_out,
                                    void* workspace, size_t workspace_bytes, nerrf_stream_t stream) {
    NERRF_REQUIRE(p && size && cost && state && actions_out && scores_out && n_out && workspace, "null pointer");
    NERRF_REQUIRE(A >= 1 && A <= 4096, "number of actions must be in 1..4096 (got %d)", A);
    NERRF_REQUIRE(n_cand >= 0 && n_cand <= 4096 && (n_cand == 0 || cand), "n_cand must be in 0..4096");
    NERRF_REQUIRE(max_commits >= 0, "negative max_commits");
    size_t need = 0;
    nerrf_plan_commit_workspace_bytes(4096, &need);
    NERRF_REQUIRE(workspace_bytes >= need && ((uintptr_t)workspace & 15) == 0, "plan-commit workspace too small or misaligned");
    cudaStream_t st = (cudaStream_t)stream;
    const int rc0 = check_cover(cover, guard, A, st);
    if (rc0) return rc0;
    unsigned char* ws = (unsigned char*)workspace;
    NERRF_CHECK_CUDA(cudaMemsetAsync(ws, 0, 256, st));
    CommitArgs a;
    a.p = p; a.size = size; a.cost = cost; a.guard = guard; a.cover = cover; a.A = A; a.state = state; a.cand = cand; a.n_cand = n_cand;
    a.max_commits = max_commits; a.allow_tentative = allow_tentative; a.cur = cur; a.cap = 4096;
    a.barrier = (unsigned*)ws;
    a.sc_buf = (float*)(ws + 256); a.flag_buf = (int32_t*)(ws + 256 + (size_t)2 * 4096 * 4);
    a.actions_out = actions_out; a.scores_out = scores_out; a.n_out = n_out;
    const int NW = nw_for(A);
    int grid = (n_cand + 7) / 8;
    if (grid < 1) grid = 1;
    if (grid > sm_count()) grid = sm_count();
    void* kargs[] = {(void*)&a};
    auto go = [&](auto kern, size_t smem) -> int {
        const int rc = set_max_dynamic_smem((const void*)kern, smem);
        if (rc) return rc;
        NERRF_CHECK_CUDA(cudaLaunchCooperativeKernel((void*)kern, dim3(grid), dim3(256), kargs, smem, st));
        return NERRF_OK;
    };
    if (NW == 1) return go(plan_commit_kernel<1>, terms_smem_bytes<1>() + 4096 * 4 + (cover ? cover_smem_bytes<1>() : 0));
    if (NW == 2) return go(plan_commit_kernel<2>, terms_smem_bytes<2>() + 4096 * 4 + (cover ? cover_smem_bytes<2>() : 0));
    return go(plan_commit_kernel<4>, terms_smem_bytes<4>() + 4096 * 4 + (cover ? cover_smem_bytes<4>() : 0));
}

extern "C" int nerrf_plan_commit(const float* p, const float* size, const float* cost, const int32_t* guard, int A,
                                 uint32_t* state, const int32_t* cand, int n_cand, float cur, int max_commits,
                                 int allow_tentative, int32_t* actions_out, float* scores_out, int32_t* n_out,
                                 void* workspace, size_t workspace_bytes, nerrf_stream_t stream) {
    return nerrf_plan_commit_ex(p, size, cost, guard, nullptr, A, state, cand, n_cand, cur, max_commits, allow_tentative,
                                actions_out, scores_out, n_out, workspace, workspace_bytes, stream);
}
