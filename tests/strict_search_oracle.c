/*
 * TEST INFRASTRUCTURE.  The search specification for both rule sets, built into one library together with tests/strict_oracle.c
 * (so_strict_moves: strict legality by its brute-force definition, sharing nothing with the bitboard attack test of cz_rules.cuh).
 *
 * Reference rules: the trees of oracle/cchess_oracle.c, compiled into this file unchanged (co_tree_search at search_threads = 1,
 * co_tree_search_fifo for search_threads = K, co_tree_search_multi for the leaf-parallel schedule).
 *
 * Strict rules (engines created with CZ_RULES_STRICT, csrc/cz_engine.cu: k_wave<T, true>): the one-leaf search restated serially
 * over the same tree.  The reference has no strict rules, so it cannot be the specification here; this file is.  It follows the
 * oracle's one-leaf search (co_tree_search: MCTS_tree.main with search_threads = 1) step for step and differs only where the rules do:
 *   expansion  the children are the strictly legal subset of the pseudo-legal list (its first 128 entries), in the same order, each
 *              with its label (flipped for black) and prior, by the reference's expansion body (expand_moves): by default tot_p =
 *              1e-8 + the serial float32 sum over these children, P /= tot_p.
 *              A position without a strictly legal move (checkmate or stalemate) is expanded with no children: it is mated.
 *   mated leaf the playout that expanded it backs up as if the network had returned -1 for the side to move there (+1 to the edge
 *              into it); the network was evaluated on it all the same.
 *   descent    after a move, in this order: a king captured, restrict_round >= 60 (both as in the reference), a child that is expanded
 *              without children (mated: +1 to the edge into it, no network call), an unexpanded child (a leaf).
 *   root       a root expanded without children is not searched.
 * Signature records carry n_children = -1 for a node expanded without children.
 *
 * Root exploration noise, for either rule set: search with 0 playouts (expands the root, runs none), replace the root priors by the
 * noised ones (rn_set_root_P; computed by the caller with numpy), search with the playouts.
 *
 * Softmax priors (engines with CZ_PRIORS_SOFTMAX, DESIGN 3k), for either rule set and every schedule: pz_tree_softmax sets the tree's
 * prior rule to pz_softmax, which the one expansion body (expand_moves) then applies to every node it expands.  pz_softmax is the
 * definition: m = the largest l_i (NaNs ignored, fmaxf), e_i = cz_exp(f64(l_i) - f64(m)), s = the f64 sum of the e_i in move order,
 * P_i = f32(e_i / s); cz_exp is the library's own header (csrc/cz_exp.h).  pz_search_shifted is the one-leaf reference search over
 * a stand-in net with a constant added to every logit (shift invariance).
 */
#include "../oracle/cchess_oracle.c"
#include "../cchess_zero_b200/csrc/cz_exp.h"

int so_strict_moves(const uint8_t *b, int side, uint16_t *moves, uint8_t *legal);

/* A strict-rules tree: a co_tree (first member, so the co_tree_* functions take it as it is) and the children its expansions made */
typedef struct {
    co_tree t;
    long sum_C;
} ss_tree;

ss_tree *ss_tree_new(const uint8_t *board) {
    ss_tree *s = (ss_tree *)calloc(1, sizeof(ss_tree));
    s->t.root = new_root(board);
    ensure_labels();
    return s;
}

/* leaf_node.expand over the strictly legal moves (error 16 and sum_C are the strict expansion's own) */
static void ss_expand(ss_tree *s, co_node *n, int side, const float *logits) {
    uint16_t mv[512];
    uint8_t ok[512];
    int c = so_strict_moves(n->board, side, mv, ok);
    if (c > MAXMOVES) { s->t.error |= 16; c = MAXMOVES; }     /* as the engine: CZ_ERR_CHILDREN, the first 128 moves are kept */
    int m = 0;
    for (int i = 0; i < c; i++)
        if (ok[i]) mv[m++] = mv[i];
    expand_moves(&s->t, n, side, logits, mv, m);
    s->sum_C += m;
}

/* one playout from the expanded root (which has children) */
static void ss_playout(ss_tree *s, int side, int rr, int net) {
    co_tree *t = &s->t;
    float x[1260], logits[NLABEL], value;
    co_node *node = t->root;
    t->plen = 0;
    for (;;) {
        double sq = sqrt((double)node->N);
        int best = 0;
        double bests = 0;
        for (int i = 0; i < node->nchild; i++) {
            co_node *c = &node->child[i];
            float p5 = 5.0f * c->P;
            double U = (double)p5 * sq / (double)(1 + c->N);
            double sc = (double)c->Q + U;
            if (i == 0 || sc > bests) { best = i; bests = sc; }
        }
        co_node *c = &node->child[best];
        t->sum_L++;
        t->sum_c += node->nchild;
        side ^= 1;
        if (count_pieces(node->board) - count_pieces(c->board) == 0) rr += 1; else rr = 0;
        c->N += 3;
        c->W = c->W - 3.0f;
        if (t->plen >= 1024) { t->error |= 4; backup_path(t, 0.0f); return; }
        t->path[t->plen++] = c;
        int hasK = has_piece(c->board, RK), hask = has_piece(c->board, BK);
        if (!hasK || !hask) {
            float v = 0;
            if (!hasK) v = (side == 1) ? 1.0f : -1.0f;
            if (!hask) v = (side == 1) ? -1.0f : 1.0f;
            backup_path(t, v * -1.0f);
            return;
        }
        if (rr >= 60) { backup_path(t, 0.0f); return; }
        if (c->expanded && c->nchild == 0) { backup_path(t, 1.0f); return; }     /* mated */
        if (!c->expanded) {                                                     /* leaf */
            co_encode(c->board, side, x);
            co_fake_forward(net, x, logits, &value);
            ss_expand(s, c, side, logits);
            backup_path(t, c->nchild == 0 ? 1.0f : -value);
            return;
        }
        node = c;
    }
}

int ss_tree_search_fake(ss_tree *s, int side, int rr, int playouts, int net) {
    co_tree *t = &s->t;
    float x[1260], logits[NLABEL], value;
    if (!t->root->expanded) {
        co_encode(t->root->board, side, x);
        co_fake_forward(net, x, logits, &value);
        ss_expand(s, t->root, side, logits);
    }
    if (t->root->nchild == 0) return t->error;
    for (int p = 0; p < playouts; p++) ss_playout(s, side, rr, net);
    return t->error;
}

/* 1 when the root is expanded without children (mated) */
int ss_tree_root_mated(ss_tree *s) { return s->t.root->expanded && s->t.root->nchild == 0; }

void ss_tree_stats(ss_tree *s, long *out) {
    co_tree *t = &s->t;
    out[0] = t->n_expand; out[1] = t->n_playout; out[2] = t->sum_L; out[3] = t->sum_c; out[4] = s->sum_C; out[5] = t->error;
}

/* co_tree_signature's records, with n_children = -1 for a node expanded without children: the same depth-first walk */
static long mark_mated(co_node *n, int64_t *out, long cap, long k) {
    for (int i = 0; i < n->nchild; i++) {
        co_node *c = &n->child[i];
        if (k < cap && c->expanded && c->nchild == 0) out[6 * k + 5] = -1;
        k++;
        if (c->expanded && c->nchild) k = mark_mated(c, out, cap, k);
    }
    return k;
}
long ss_tree_signature(ss_tree *s, int64_t *out, long cap) {
    long k = co_tree_signature(&s->t, out, cap);
    mark_mated(s->t.root, out, cap, 0);
    return k;
}

/* Root priors <- P[0 .. n) of an expanded root, for either rule set; -1 (nothing changed) when the root is not expanded. */
int rn_set_root_P(co_tree *t, const float *P) {
    co_node *r = t->root;
    if (!r->expanded) return -1;
    for (int i = 0; i < r->nchild; i++) r->child[i].P = P[i];
    return 0;
}

/* Softmax priors, in place on the logits P[0 .. n) of one node's children (n at most expand_moves' MAXMOVES + 8) */
void pz_softmax(float *P, int n) {
    double e[MAXMOVES + 8];
    if (n < 1) return;
    float m = P[0];
    for (int i = 1; i < n; i++) m = fmaxf(m, P[i]);
    double s = 0.0;
    for (int i = 0; i < n; i++) {
        e[i] = cz_exp((double)P[i] - (double)m);
        s = s + e[i];
    }
    for (int i = 0; i < n; i++) P[i] = (float)(e[i] / s);
}

/* Every later expansion of the tree (either rule set, every schedule) uses softmax priors */
void pz_tree_softmax(co_tree *t) { t->priors = pz_softmax; }

void pz_exp(const double *x, double *y, long n) {
    for (long i = 0; i < n; i++) y[i] = cz_exp(x[i]);
}

/* co_tree_search (reference rules, one leaf) over the stand-in net `net` with `shift` added to every logit (f32 adds; exact on the
 * stand-ins' grids for shift = 1) */
typedef struct { int net; float shift; } pz_net;
static void pz_forward(void *ctx, const float *x, float *logits, float *value) {
    const pz_net *p = (const pz_net *)ctx;
    co_fake_forward(p->net, x, logits, value);
    for (int i = 0; i < NLABEL; i++) logits[i] = logits[i] + p->shift;
}
int pz_search_shifted(co_tree *t, int side, int rr, int playouts, int net, float shift) {
    pz_net nt = {net, shift};
    return co_tree_search(t, side, rr, playouts, pz_forward, &nt);
}
