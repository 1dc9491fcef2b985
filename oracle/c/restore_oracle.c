/* planner spec v2 oracle in plain C  --  TEST INFRASTRUCTURE (see oracle/__init__.py): a second, independent restatement
 * of oracle/restore_ref.py (rewards with cover / "restore from backup" actions, DESIGN.md 1.3; reference prose:
 * threat-model.mdx:205-223, architecture.mdx:104-108) and of the leaf-parallel search that uses it.
 *
 * Build: gcc -O2 -fopenmp -ffp-contract=off -fno-fast-math -shared -fPIC   (every fp32 op individually rounded).
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

static void philox(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3, uint32_t k0, uint32_t k1, uint32_t out[4]) {
    const uint32_t M0 = 0xD2511F53u, M1 = 0xCD9E8D57u, W0 = 0x9E3779B9u, W1 = 0xBB67AE85u;
    for (int r = 0; r < 10; ++r) {
        const uint64_t p0 = (uint64_t)M0 * c0, p1 = (uint64_t)M1 * c2;
        const uint32_t n0 = (uint32_t)(p1 >> 32) ^ c1 ^ k0, n2 = (uint32_t)(p0 >> 32) ^ c3 ^ k1;
        c1 = (uint32_t)p1; c3 = (uint32_t)p0; c0 = n0; c2 = n2;
        k0 += W0; k1 += W1;
    }
    out[0] = c0; out[1] = c1; out[2] = c2; out[3] = c3;
}

typedef struct {
    int chunk, A_pad, n_words;
    float *u, *v, *vw, *c;   /* [A_pad]; vw = v + p_guard * u where a guard exists, else v */
    int *g, *cv;             /* [A_pad] guard / cover index or -1 */
} V2;

static void v2_init(V2* t, const float* p, const float* size, const float* cost, const int32_t* guard,
                    const int32_t* cover, int A) {
    const int NW = A <= 1024 ? 1 : (A <= 2048 ? 2 : 4);
    t->chunk = 32 * NW; t->A_pad = 1024 * NW; t->n_words = 32 * NW;
    t->u = (float*)calloc(t->A_pad, 4); t->v = (float*)calloc(t->A_pad, 4);
    t->vw = (float*)calloc(t->A_pad, 4); t->c = (float*)calloc(t->A_pad, 4);
    t->g = (int*)malloc(t->A_pad * sizeof(int)); t->cv = (int*)malloc(t->A_pad * sizeof(int));
    for (int a = 0; a < t->A_pad; ++a) { t->g[a] = -1; t->cv[a] = -1; }
    for (int a = 0; a < A; ++a) {
        const float u = p[a] * size[a];
        const float one_minus = 1.0f - p[a];
        const float v = one_minus * size[a];
        t->u[a] = u; t->v[a] = v; t->vw[a] = v; t->c[a] = cost[a];
        if (guard && guard[a] >= 0) {
            t->g[a] = guard[a];
            const float w = p[guard[a]] * u;
            t->vw[a] = v + w;
        }
        if (cover && cover[a] >= 0) t->cv[a] = cover[a];
    }
}
static void v2_free(V2* t) { free(t->u); free(t->v); free(t->vw); free(t->c); free(t->g); free(t->cv); }

static int bit(const uint32_t* s, int a) { return (int)((s[a >> 5] >> (a & 31)) & 1u); }

static float v2_score(const V2* t, const uint32_t* s) {
    float dl[32], dt[32];
    for (int l = 0; l < 32; ++l) {
        float x = 0.f, y = 0.f;
        for (int i = 0; i < t->chunk; ++i) {
            const int a = l * t->chunk + i;
            const int in_s = bit(s, a);
            const int restored = in_s || (t->cv[a] >= 0 && bit(s, t->cv[a]));
            const int alive = t->g[a] >= 0 && !bit(s, t->g[a]);
            float term;
            if (restored) term = alive ? t->vw[a] : t->v[a];
            else term = t->u[a];
            x = x + term;
            y = y + (in_s ? t->c[a] : 0.f);
        }
        dl[l] = x; dt[l] = y;
    }
    for (int st = 1; st < 32; st <<= 1) {
        float nl[32], nt[32];
        for (int l = 0; l < 32; ++l) { nl[l] = dl[l] + dl[l ^ st]; nt[l] = dt[l] + dt[l ^ st]; }
        memcpy(dl, nl, sizeof(dl)); memcpy(dt, nt, sizeof(dt));
    }
    const float tenth = 0.1f * dt[0];
    return -(dl[0] + tenth);
}

void nerrf_oracle_v2_score(const uint32_t* states, int64_t B, const float* p, const float* size, const float* cost,
                           const int32_t* guard, const int32_t* cover, int A, float* out) {
    V2 t; v2_init(&t, p, size, cost, guard, cover, A);
#pragma omp parallel for schedule(static)
    for (int64_t b = 0; b < B; ++b) out[b] = v2_score(&t, states + b * t.n_words);
    v2_free(&t);
}

static int zeros(const uint32_t* s, int nw) { int z = 0; for (int k = 0; k < nw; ++k) z += __builtin_popcount(~s[k]); return z; }
static int jth_zero(const uint32_t* s, int nw, int j) {
    for (int a = 0; a < 32 * nw; ++a)
        if (!bit(s, a)) { if (j == 0) return a; --j; }
    return -1;
}

/* leaf-parallel UCT as oracle/mcts_ref.py, valued with the spec-v2 reward.  root_n / root_w [A_pad] out. */
int nerrf_oracle_v2_mcts(const float* p, const float* size, const float* cost, const int32_t* guard, const int32_t* cover,
                         int A, const uint32_t* root_state, int R, int D, int T, uint64_t seed, float c, float lo,
                         float inv_range, const float* lnN, int32_t* root_n, float* root_w, int32_t* num_nodes_out) {
    V2 t; v2_init(&t, p, size, cost, guard, cover, A);
    const int nw = t.n_words, Ap = t.A_pad;
    const uint32_t k0 = (uint32_t)seed, k1 = (uint32_t)(seed >> 32);
    const size_t cells = (size_t)(T + 1) * Ap;
    int32_t* visits = (int32_t*)calloc(T + 1, 4);
    int32_t* cn = (int32_t*)calloc(cells, 4);
    float* cw = (float*)calloc(cells, 4);
    int32_t* cid = (int32_t*)malloc(cells * 4);
    for (size_t i = 0; i < cells; ++i) cid[i] = -1;
    float* val = (float*)malloc((size_t)R * 4);
    uint32_t* root = (uint32_t*)malloc(nw * 4);
    uint32_t* state = (uint32_t*)malloc(nw * 4);
    int* pn = (int*)malloc((D + 2) * sizeof(int));
    int* pa = (int*)malloc((D + 2) * sizeof(int));
    for (int k = 0; k < nw; ++k) root[k] = root_state ? root_state[k] : 0u;
    for (int a = A; a < Ap; ++a) root[a >> 5] |= 1u << (a & 31);
    int num_nodes = 1;
    for (int it = 0; it < T; ++it) {
        int node = 0, depth = 0, plen = 0;
        memcpy(state, root, nw * 4);
        while (visits[node] > 0 && depth < D && zeros(state, nw) > 0) {
            float best = -INFINITY;
            int ba = -1;
            for (int a = 0; a < Ap; ++a) {
                if (bit(state, a)) continue;
                const int n = cn[(size_t)node * Ap + a];
                float key = INFINITY;
                if (n > 0) {
                    const float nf = (float)n;
                    const float q = cw[(size_t)node * Ap + a] / nf;
                    const float r = lnN[visits[node]] / nf;
                    const float e = c * sqrtf(r);
                    key = q + e;
                }
                if (key > best) { best = key; ba = a; }
            }
            pn[plen] = node; pa[plen] = ba; ++plen;
            state[ba >> 5] |= 1u << (ba & 31);
            ++depth;
            const int child = cid[(size_t)node * Ap + ba];
            if (child < 0) { cid[(size_t)node * Ap + ba] = num_nodes; node = num_nodes++; break; }
            node = child;
        }
        const int leaf = node, L0 = zeros(state, nw), first = (D - depth) > 0 && L0 > 0;
#pragma omp parallel
        {
            uint32_t* s = (uint32_t*)malloc(nw * 4);
#pragma omp for schedule(static)
            for (int r = 0; r < R; ++r) {
                memcpy(s, state, nw * 4);
                int left = D - depth, L = L0;
                if (first) { const int a = jth_zero(s, nw, r % L0); s[a >> 5] |= 1u << (a & 31); --left; --L; }
                uint32_t rnd[4] = {0, 0, 0, 0};
                for (int k = 0; k < left && L > 0; ++k, --L) {
                    if ((k & 3) == 0) philox((uint32_t)r, (uint32_t)(k >> 2), (uint32_t)it, 0u, k0, k1, rnd);
                    const int a = jth_zero(s, nw, (int)(((uint64_t)rnd[k & 3] * (uint32_t)L) >> 32));
                    s[a >> 5] |= 1u << (a & 31);
                }
                const float d = v2_score(&t, s) - lo;
                val[r] = d * inv_range;
            }
            free(s);
        }
        if (first) {
            for (int q = 0; q < (R < L0 ? R : L0); ++q) {
                const size_t idx = (size_t)leaf * Ap + jth_zero(state, nw, q);
                for (int r = q; r < R; r += L0) { cw[idx] = cw[idx] + val[r]; ++cn[idx]; }
            }
        }
        for (int n = R; n > 1; n >>= 1)                   /* adjacent-pairs tree sum, in place */
            for (int i = 0; i < n / 2; ++i) val[i] = val[2 * i] + val[2 * i + 1];
        visits[leaf] += 1;
        for (int i = 0; i < plen; ++i) {
            const size_t idx = (size_t)pn[i] * Ap + pa[i];
            cn[idx] += R;
            cw[idx] = cw[idx] + val[0];
            visits[pn[i]] += 1;
        }
    }
    memcpy(root_n, cn, (size_t)Ap * 4);
    memcpy(root_w, cw, (size_t)Ap * 4);
    *num_nodes_out = num_nodes;
    free(visits); free(cn); free(cw); free(cid); free(val); free(root); free(state); free(pn); free(pa); v2_free(&t);
    return 0;
}
