// cz_host.cu -- host-side move choice for thousands of games per ply: get_action's sampling (main.py:1339-1348) for the whole batch
// in native code, bit-identical to the numpy calls the reference makes.
//
// The reference draws, per move:  p = 0.75 * probs + 0.25 * np.random.dirichlet(0.3 * ones(n));  act = np.random.choice(actions, p=p)
// on numpy's legacy global RandomState (MT19937).  With thousands of concurrent games a Python loop over games costs ~25 us per game
// and ply (5 % of a step at 1024 games); this file restates exactly what those numpy calls compute -- same generator, same
// algorithms, same floating-point operation order -- so the draws, the chosen moves and the recorded pi are bit-identical:
//   probs      = ex / np.sum(ex)                      numpy pairwise summation (8 accumulators, <= 128 elements: one block)
//   dirichlet  = legacy_standard_gamma(0.3) per element (Ahrens-Dieter rejection, shape < 1) then * (1 / sum)      [mtrand.pyx dirichlet]
//   choice     = cdf = cumsum(p); cdf /= cdf[-1]; searchsorted(cdf, random_sample(), side='right')                    [mtrand.pyx choice]
//   MT19937    = genrand_int32; random_sample = ((a >> 5) * 67108864 + (b >> 6)) / 9007199254740992
// One generator state per game slot (SelfPlay's per-game RandomState), exported from / importable into numpy.RandomState.
// cz_host_dirichlet draws RandomState.dirichlet(alpha * ones(n)) the same way for SelfPlay's root exploration noise (any 0 < alpha < 1).
// Host code only (built by nvcc's host compiler with -ffp-contract=off: every operation is one IEEE operation).
#include <math.h>
#include <stdint.h>
#include <string.h>

#include <thread>
#include <vector>

#include "../../include/cchess_b200.h"

namespace {

struct MT {
    uint32_t key[624];
    uint32_t pos;
    uint32_t pad;
};
static_assert(sizeof(MT) == CZ_MT_WORDS * 4, "state layout");

inline uint32_t mt_next(MT &s) {
    if (s.pos == 624) {   // mt19937_gen: regenerate the block
        int i;
        uint32_t y;
        const uint32_t N = 624, M = 397, MATRIX_A = 0x9908b0dfu, UPPER = 0x80000000u, LOWER = 0x7fffffffu;
        for (i = 0; i < (int)(N - M); i++) {
            y = (s.key[i] & UPPER) | (s.key[i + 1] & LOWER);
            s.key[i] = s.key[i + M] ^ (y >> 1) ^ (-(int32_t)(y & 1) & MATRIX_A);
        }
        for (; i < (int)N - 1; i++) {
            y = (s.key[i] & UPPER) | (s.key[i + 1] & LOWER);
            s.key[i] = s.key[i + (M - N)] ^ (y >> 1) ^ (-(int32_t)(y & 1) & MATRIX_A);
        }
        y = (s.key[N - 1] & UPPER) | (s.key[0] & LOWER);
        s.key[N - 1] = s.key[M - 1] ^ (y >> 1) ^ (-(int32_t)(y & 1) & MATRIX_A);
        s.pos = 0;
    }
    uint32_t y = s.key[s.pos++];
    y ^= (y >> 11);
    y ^= (y << 7) & 0x9d2c5680u;
    y ^= (y << 15) & 0xefc60000u;
    y ^= (y >> 18);
    return y;
}
inline double mt_double(MT &s) {
    const int32_t a = (int32_t)(mt_next(s) >> 5), b = (int32_t)(mt_next(s) >> 6);
    return (a * 67108864.0 + b) / 9007199254740992.0;
}
inline double legacy_exponential(MT &s) { return -log(1.0 - mt_double(s)); }
// numpy/random/src/legacy/legacy-distributions.c: legacy_standard_gamma, branch shape < 1
inline double legacy_gamma_lt1(MT &s, double shape) {
    for (;;) {
        const double U = mt_double(s);
        const double V = legacy_exponential(s);
        if (U <= 1.0 - shape) {
            const double X = pow(U, 1. / shape);
            if (X <= V) return X;
        } else {
            const double Y = -log((1 - U) / shape);
            const double X = pow(1.0 - shape + shape * Y, 1. / shape);
            if (X <= (V + Y)) return X;
        }
    }
}
// numpy/core/src/umath/loops_utils.h: DOUBLE_pairwise_sum for n <= 128 (one block)
inline double pairwise_sum(const double *a, int n) {
    if (n < 8) {
        double res = 0.;
        for (int i = 0; i < n; i++) res += a[i];
        return res;
    }
    double r[8];
    for (int j = 0; j < 8; j++) r[j] = a[j];
    int i;
    for (i = 8; i < n - (n % 8); i += 8)
        for (int j = 0; j < 8; j++) r[j] += a[i + j];
    double res = ((r[0] + r[1]) + (r[2] + r[3])) + ((r[4] + r[5]) + (r[6] + r[7]));
    for (; i < n; i++) res += a[i];
    return res;
}
// RandomState.dirichlet(alpha * ones(n)) for 0 < alpha < 1 [mtrand.pyx dirichlet]: n gamma draws in order, their serial sum, then
// each scaled by 1 / sum
inline void dirichlet_lt1(MT &s, double alpha, int n, double *d) {
    double acc = 0.0;
    for (int j = 0; j < n; j++) { d[j] = legacy_gamma_lt1(s, alpha); acc = acc + d[j]; }
    const double invacc = 1 / acc;
    for (int j = 0; j < n; j++) d[j] = d[j] * invacc;
}

void choose_range(int g0, int g1, const uint8_t *live, const int32_t *n_children, const double *ex, int exploration, MT *mt,
                  int32_t *choice, double *probs, uint8_t *fallback) {
    double d[CZ_MAXCHILD], cdf[CZ_MAXCHILD];
    for (int g = g0; g < g1; g++) {
        choice[g] = -1;
        fallback[g] = 0;
        if (live && !live[g]) continue;
        const int n = n_children[g];
        if (n <= 0 || n > CZ_MAXCHILD) { fallback[g] = 1; continue; }
        const double *e = ex + (size_t)g * CZ_MAXCHILD;
        double *p = probs + (size_t)g * CZ_MAXCHILD;
        const double tot = 0.0 + pairwise_sum(e, n);                 // np.sum(probs): add.reduce starts from the identity
        for (int i = 0; i < n; i++) p[i] = e[i] / tot;               // probs /= np.sum(probs)
        const double *q = p;
        if (exploration) {
            // validity of the mixed vector is checked before any draw is consumed? No: numpy draws the Dirichlet first (argument
            // evaluation), then choice() validates p.  Mirror that order.
            dirichlet_lt1(mt[g], 0.3, n, d);
            for (int j = 0; j < n; j++) cdf[j] = 0.75 * p[j] + 0.25 * d[j];   // the mixed p (held in cdf[] until the cumsum below)
            q = cdf;
        }
        // np.random.choice(actions, p=q): the caller falls back to numpy itself whenever q would make numpy raise
        bool bad = false;
        double minv = q[0];
        for (int j = 0; j < n; j++) { if (!(q[j] == q[j])) bad = true; if (q[j] < minv) minv = q[j]; }
        double c = 0.0;
        for (int j = 0; j < n; j++) { c = c + q[j]; cdf[j] = c; }             // p.cumsum()
        const double last = cdf[n - 1];
        if (bad || !(last == last) || fabs(last - 1.0) > 1.5e-8 * (n > 1 ? (double)n : 1.0) || minv < 0) { fallback[g] = 1; continue; }
        for (int j = 0; j < n; j++) cdf[j] = cdf[j] / last;                   // cdf /= cdf[-1]
        const double u = mt_double(mt[g]);                                    // random_sample()
        int lo = 0, hi = n;                                                   // searchsorted(side='right'): first index with cdf > u
        while (lo < hi) { const int mid = (lo + hi) >> 1; if (cdf[mid] <= u) lo = mid + 1; else hi = mid; }
        choice[g] = lo;
    }
}

void dirichlet_range(int g0, int g1, const uint8_t *mask, const int32_t *n, double alpha, MT *mt, double *eta) {
    for (int g = g0; g < g1; g++)
        if ((!mask || mask[g]) && n[g] > 0) dirichlet_lt1(mt[g], alpha, n[g], eta + (size_t)g * CZ_MAXCHILD);
}

// run(g0, g1) over n_threads contiguous ranges of games, one thread each (at least 32 games per thread; one range runs on the caller)
template <typename F>
void over_games(int n_games, int n_threads, F run) {
    if (n_threads < 1) n_threads = 1;
    if (n_threads > n_games / 32) n_threads = n_games / 32 > 0 ? n_games / 32 : 1;
    if (n_threads == 1) { run(0, n_games); return; }
    std::vector<std::thread> th;
    const int per = (n_games + n_threads - 1) / n_threads;
    for (int t = 0; t < n_threads; t++) {
        const int g0 = t * per, g1 = g0 + per < n_games ? g0 + per : n_games;
        if (g0 >= g1) break;
        th.emplace_back(run, g0, g1);
    }
    for (auto &t : th) t.join();
}

}  // namespace

extern "C" {

int cz_host_choose_moves(int n_games, const uint8_t *live, const int32_t *n_children, const double *ex, int exploration, uint32_t *mt_states,
                         int32_t *choice, double *probs, uint8_t *fallback, int n_threads) {
    if (n_games < 0 || !n_children || !ex || !mt_states || !choice || !probs || !fallback) return CZ_EINVAL;
    MT *mt = reinterpret_cast<MT *>(mt_states);
    over_games(n_games, n_threads, [=](int g0, int g1) { choose_range(g0, g1, live, n_children, ex, exploration, mt, choice, probs, fallback); });
    return CZ_OK;
}

int cz_host_dirichlet(int n_games, const uint8_t *mask, const int32_t *n, const double *alpha_p, uint32_t *mt_states, double *eta, int n_threads) {
    if (n_games < 0 || !n || !alpha_p || !mt_states || !eta) return CZ_EINVAL;
    const double alpha = *alpha_p;
    if (!(alpha > 0.0 && alpha < 1.0)) return CZ_EINVAL;
    for (int g = 0; g < n_games; g++)
        if ((!mask || mask[g]) && n[g] > CZ_MAXCHILD) return CZ_EINVAL;
    MT *mt = reinterpret_cast<MT *>(mt_states);
    over_games(n_games, n_threads, [=](int g0, int g1) { dirichlet_range(g0, g1, mask, n, alpha, mt, eta); });
    return CZ_OK;
}

}  // extern "C"
