/*
 * TEST INFRASTRUCTURE.  Root exploration noise in the C specification trees: the reference-rules tree of oracle/cchess_oracle.c
 * (co_tree_search at K = 1, co_tree_search_fifo at K = 16), compiled into this file unchanged, plus a setter for the root priors.
 * A noisy search is then: search with 0 playouts (expands the root, runs none), replace the root priors by the noised ones
 * (computed by the caller with numpy), search with the playouts.  Built together with tests/root_noise_strict_oracle.c (the same
 * setter for the strict-rules tree) and tests/strict_oracle.c.
 */
#include "../oracle/cchess_oracle.c"

/* Root priors <- P[0 .. n) of an expanded root; -1 (nothing changed) when the root is not expanded. */
int rn_co_set_root_P(co_tree *t, const float *P) {
    co_node *r = t->root;
    if (!r->expanded) return -1;
    for (int i = 0; i < r->nchild; i++) r->child[i].P = P[i];
    return 0;
}
