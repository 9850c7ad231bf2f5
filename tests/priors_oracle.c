/*
 * TEST INFRASTRUCTURE.  Softmax priors (engines with CZ_PRIORS_SOFTMAX, DESIGN 3k) over the search specification of
 * tests/strict_search_oracle.c (both rule sets), which is compiled into this file unchanged.
 *
 *   pz_softmax  the definition for one node: m = the largest l_i (NaNs ignored, fmaxf), e_i = cz_exp(f64(l_i) - f64(m)), s = the
 *               f64 sum of the e_i in move order, P_i = f32(e_i / s).  cz_exp is the library's own header (csrc/cz_exp.h).
 *   pz_search   a one-leaf search with softmax priors.  The specification's expansions write the reference priors; after the root
 *               expansion and after every playout, each node expanded since then gets its priors replaced by pz_softmax of the
 *               same logits (the stand-in net evaluated on the node again, the same children and label indices as the expansion).
 *               A one-leaf playout reads no prior of the node it expands, so this is the search that expands with softmax priors.
 *               The K-coroutine and leaf-parallel schedules do read them within one call; they are not covered here.
 * A node whose priors have been replaced carries inflight = -1 (a field only the leaf-parallel specification uses).
 */
#include "strict_search_oracle.c"
#include "../cchess_zero_b200/csrc/cz_exp.h"

/* P[0 .. n) from the logits l[0 .. n), n <= 128; returns -1 (nothing written) for another n */
int pz_softmax(const float *l, int n, float *P) {
    double e[MAXMOVES];
    if (n < 1 || n > MAXMOVES) return -1;
    float m = l[0];
    for (int i = 1; i < n; i++) m = fmaxf(m, l[i]);
    double s = 0.0;
    for (int i = 0; i < n; i++) {
        e[i] = cz_exp((double)l[i] - (double)m);
        s = s + e[i];
    }
    for (int i = 0; i < n; i++) P[i] = (float)(e[i] / s);
    return 0;
}

void pz_exp(const double *x, double *y, long n) {
    for (long i = 0; i < n; i++) y[i] = cz_exp(x[i]);
}

/* the stand-in net `net` with `shift` added to every logit (f32 adds; exact on the stand-ins' grids for shift = 1) */
typedef struct { int net; float shift; } pz_net;
static void pz_forward(void *ctx, const float *x, float *logits, float *value) {
    const pz_net *p = (const pz_net *)ctx;
    co_fake_forward(p->net, x, logits, value);
    if (p->shift != 0.0f)
        for (int i = 0; i < NLABEL; i++) logits[i] = logits[i] + p->shift;
}

/* the priors of an expanded node's children from the net's logits at (board, side), gathered as expand() gathers them */
static void pz_fix(co_tree *t, co_node *n, int side, pz_net *net) {
    float x[1260], logits[NLABEL], value, l[MAXMOVES], P[MAXMOVES];
    co_encode(n->board, side, x);
    pz_forward(net, x, logits, &value);
    for (int i = 0; i < n->nchild; i++) {
        const int mv = n->child[i].move;
        int li = g_label_of[mv & 127][mv >> 7];
        if (li < 0) { t->error |= 2; li = 0; }
        if (side == 1) li = g_unflipped[li];
        l[i] = logits[li];
    }
    if (pz_softmax(l, n->nchild, P) == 0)
        for (int i = 0; i < n->nchild; i++) n->child[i].P = P[i];
}

static void pz_walk(co_tree *t, co_node *n, int side, pz_net *net) {
    if (!n->expanded) return;
    if (n->inflight != -1) {
        if (n->nchild) pz_fix(t, n, side, net);
        n->inflight = -1;
    }
    for (int i = 0; i < n->nchild; i++) pz_walk(t, &n->child[i], side ^ 1, net);
}

static int pz_step(co_tree *t, int strict, int side, int rr, int playouts, pz_net *net) {
    if (strict) return ss_tree_search_fake((ss_tree *)t, side, rr, playouts, net->net);
    return co_tree_search(t, side, rr, playouts, pz_forward, net);
}

/* A one-leaf search: co_tree_search over the stand-in net `net` with `shift` added to its logits (strict = 0), or
 * ss_tree_search_fake (strict = 1, t an ss_tree, shift 0); softmax = 1: with softmax priors.  -1 for a shift under strict rules. */
int pz_search(co_tree *t, int strict, int side, int rr, int playouts, int net, float shift, int softmax) {
    pz_net nt = {net, shift};
    if (strict && shift != 0.0f) return -1;
    if (!softmax) return pz_step(t, strict, side, rr, playouts, &nt);
    int err = pz_step(t, strict, side, rr, 0, &nt);
    pz_walk(t, t->root, side, &nt);
    for (int p = 0; p < playouts; p++) {
        err = pz_step(t, strict, side, rr, 1, &nt);
        pz_walk(t, t->root, side, &nt);
    }
    return err;
}
