/*
 * TEST INFRASTRUCTURE.  The strict-rules specification tree (tests/strict_search_oracle.c, compiled into this file unchanged) with a
 * setter for the root priors, for the root-noise tests; see tests/root_noise_oracle.c.
 */
#include "strict_search_oracle.c"

/* Root priors <- P[0 .. n) of an expanded root; -1 (nothing changed) when the root is not expanded. */
int rn_ss_set_root_P(ss_tree *t, const float *P) {
    ss_node *r = t->root;
    if (!r->expanded) return -1;
    for (int i = 0; i < r->nchild; i++) r->child[i].P = P[i];
    return 0;
}
