/*
 * TEST INFRASTRUCTURE.  The specification of the one-leaf search under the STRICT rules (engines created with CZ_RULES_STRICT,
 * csrc/cz_engine.cu: k_wave<T, true>), restated serially in plain C.  Compiled together with oracle/cchess_oracle.c (move
 * generation, board update, encoding, stand-in nets, label tables) and tests/strict_oracle.c (so_strict_moves: strict legality by
 * its brute-force definition, sharing nothing with the bitboard attack test of cz_rules.cuh).
 *
 * The reference has no strict rules, so it cannot be the specification here; this file is.  It follows the oracle's one-leaf search
 * (co_tree_search: MCTS_tree.main with search_threads = 1) step for step and differs only where the rules do:
 *   expansion  the children are the strictly legal subset of the pseudo-legal list (its first 128 entries), in the same order, each
 *              with its label (flipped for black) and prior; tot_p = 1e-8 + the serial float32 sum over these children, P /= tot_p.
 *              A position without a strictly legal move (checkmate or stalemate) is expanded with no children: it is mated.
 *   mated leaf the playout that expanded it backs up as if the network had returned -1 for the side to move there (+1 to the edge
 *              into it); the network was evaluated on it all the same.
 *   descent    after a move, in this order: a king captured, restrict_round >= 60 (both as in the reference), a child that is expanded
 *              without children (mated: +1 to the edge into it, no network call), an unexpanded child (a leaf).
 *   root       a root expanded without children is not searched.
 * Signature records carry n_children = -1 for a node expanded without children.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

int co_legal_moves(const uint8_t *b, int side, uint16_t *out);
int co_apply_move(uint8_t *b, int mv);
void co_encode(const uint8_t *b, int side, float *out);
void co_fake_forward(int net, const float *x, float *logits, float *value);
int co_label_index(int src, int dst);
int co_unflipped_index(int i);
int so_strict_moves(const uint8_t *b, int side, uint16_t *moves, uint8_t *legal);

#define SS_NLABEL 2086
#define SS_MAXCHILD 128
#define SS_MAXPATH 1024

typedef struct ss_node {
    float P, W, Q;
    int N;
    int nchild;
    int expanded;
    uint16_t move;
    struct ss_node *child;
    uint8_t board[90];
} ss_node;

typedef struct {
    ss_node *root;
    ss_node *path[SS_MAXPATH];
    int plen;
    long n_expand, n_playout, sum_L, sum_c, sum_C;
    int error;          /* 2: move without a label, 4: path too deep, 16: more than 128 pseudo-legal moves */
} ss_tree;

static void free_children(ss_node *n) {
    if (!n->child) return;
    for (int i = 0; i < n->nchild; i++) free_children(&n->child[i]);
    free(n->child);
    n->child = NULL;
}

ss_tree *ss_tree_new(const uint8_t *board) {
    ss_tree *t = (ss_tree *)calloc(1, sizeof(ss_tree));
    t->root = (ss_node *)calloc(1, sizeof(ss_node));
    memcpy(t->root->board, board, 90);
    return t;
}

void ss_tree_free(ss_tree *t) {
    if (!t) return;
    free_children(t->root);
    free(t->root);
    free(t);
}

/* leaf_node.expand over the strictly legal moves */
static void expand(ss_tree *t, ss_node *n, int side, const float *logits) {
    uint16_t mv[512];
    uint8_t ok[512];
    int c = so_strict_moves(n->board, side, mv, ok);
    if (c > SS_MAXCHILD) { t->error |= 16; c = SS_MAXCHILD; }     /* as the engine: CZ_ERR_CHILDREN, the first 128 moves are kept */
    int m = 0;
    for (int i = 0; i < c; i++)
        if (ok[i]) mv[m++] = mv[i];
    n->child = (ss_node *)calloc(m > 0 ? m : 1, sizeof(ss_node));
    n->nchild = m;
    float tot = 1e-8f;
    for (int i = 0; i < m; i++) {
        ss_node *ch = &n->child[i];
        int li = co_label_index(mv[i] & 127, mv[i] >> 7);
        if (li < 0) { t->error |= 2; li = 0; }
        if (side == 1) li = co_unflipped_index(li);
        memcpy(ch->board, n->board, 90);
        co_apply_move(ch->board, mv[i]);
        ch->move = mv[i];
        ch->P = logits[li];
        tot = tot + ch->P;
    }
    for (int i = 0; i < m; i++) n->child[i].P = n->child[i].P / tot;
    n->expanded = 1;
    t->n_expand++;
    t->sum_C += m;
}

/* VL undo + back_up_value along the path; val is the value handed to the deepest edge */
static void backup_path(ss_tree *t, float val) {
    for (int d = t->plen - 1; d >= 0; d--) {
        ss_node *c = t->path[d];
        c->N += -3;
        c->W = c->W + 3.0f;
        c->N += 1;
        c->W = c->W + val;
        c->Q = c->W / (float)c->N;
        val = -val;
    }
    t->plen = 0;
    t->n_playout++;
}

static int has_piece(const uint8_t *b, int p) { for (int i = 0; i < 90; i++) if (b[i] == p) return 1; return 0; }
static int count_pieces(const uint8_t *b) { int c = 0; for (int i = 0; i < 90; i++) c += b[i] != 0; return c; }

/* one playout from the expanded root (which has children) */
static void playout(ss_tree *t, int side, int rr, int net) {
    float x[1260], logits[SS_NLABEL], value;
    ss_node *node = t->root;
    t->plen = 0;
    for (;;) {
        double sq = sqrt((double)node->N);
        int best = 0;
        double bests = 0;
        for (int i = 0; i < node->nchild; i++) {
            ss_node *c = &node->child[i];
            float p5 = 5.0f * c->P;
            double U = (double)p5 * sq / (double)(1 + c->N);
            double s = (double)c->Q + U;
            if (i == 0 || s > bests) { best = i; bests = s; }
        }
        ss_node *c = &node->child[best];
        t->sum_L++;
        t->sum_c += node->nchild;
        side ^= 1;
        if (count_pieces(node->board) - count_pieces(c->board) == 0) rr += 1; else rr = 0;
        c->N += 3;
        c->W = c->W - 3.0f;
        if (t->plen >= SS_MAXPATH) { t->error |= 4; backup_path(t, 0.0f); return; }
        t->path[t->plen++] = c;
        int hasK = has_piece(c->board, 1), hask = has_piece(c->board, 8);
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
            expand(t, c, side, logits);
            backup_path(t, c->nchild == 0 ? 1.0f : -value);
            return;
        }
        node = c;
    }
}

int ss_tree_search_fake(ss_tree *t, int side, int rr, int playouts, int net) {
    float x[1260], logits[SS_NLABEL], value;
    if (!t->root->expanded) {
        co_encode(t->root->board, side, x);
        co_fake_forward(net, x, logits, &value);
        expand(t, t->root, side, logits);
    }
    if (t->root->nchild == 0) return t->error;
    for (int p = 0; p < playouts; p++) playout(t, side, rr, net);
    return t->error;
}

/* root children in order; -1 when the root is not expanded */
int ss_tree_root_children(ss_tree *t, uint16_t *moves, int *N, float *W, float *P, float *Q) {
    ss_node *r = t->root;
    for (int i = 0; i < r->nchild; i++) {
        ss_node *c = &r->child[i];
        moves[i] = c->move; N[i] = c->N; W[i] = c->W; P[i] = c->P; Q[i] = c->Q;
    }
    return r->expanded ? r->nchild : -1;
}

/* re-root on child idx, keeping its subtree */
int ss_tree_update(ss_tree *t, int idx) {
    ss_node *r = t->root;
    if (idx < 0 || idx >= r->nchild) return -1;
    ss_node *nr = (ss_node *)malloc(sizeof(ss_node));
    *nr = r->child[idx];
    for (int i = 0; i < r->nchild; i++) if (i != idx) free_children(&r->child[i]);
    free(r->child);
    free(r);
    t->root = nr;
    return 0;
}

/* 1 when the root is expanded without children (mated) */
int ss_tree_root_mated(ss_tree *t) { return t->root->expanded && t->root->nchild == 0; }

void ss_tree_stats(ss_tree *t, long *out) {
    out[0] = t->n_expand; out[1] = t->n_playout; out[2] = t->sum_L; out[3] = t->sum_c; out[4] = t->sum_C; out[5] = t->error;
}

/* (label index, N, W bits, P bits, Q bits, n_children: -1 expanded without children, 0 not expanded) in depth-first order */
static long sig_rec(ss_node *n, int64_t *out, long cap, long k) {
    for (int i = 0; i < n->nchild; i++) {
        ss_node *c = &n->child[i];
        if (k < cap) {
            uint32_t w, p, q;
            memcpy(&w, &c->W, 4); memcpy(&p, &c->P, 4); memcpy(&q, &c->Q, 4);
            if (c->W != c->W) w = 0x7FC00000u;
            if (c->P != c->P) p = 0x7FC00000u;
            if (c->Q != c->Q) q = 0x7FC00000u;
            int64_t *r = out + 6 * k;
            r[0] = co_label_index(c->move & 127, c->move >> 7); r[1] = c->N; r[2] = w; r[3] = p; r[4] = q;
            r[5] = c->expanded ? (c->nchild ? c->nchild : -1) : 0;
        }
        k++;
        if (c->expanded && c->nchild) k = sig_rec(c, out, cap, k);
    }
    return k;
}
long ss_tree_signature(ss_tree *t, int64_t *out, long cap) { return sig_rec(t->root, out, cap, 0); }
