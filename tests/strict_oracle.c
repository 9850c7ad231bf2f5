/*
 * TEST INFRASTRUCTURE.  Strict legality by its definition, the slow way, over the parity oracle's move generator
 * (oracle/cchess_oracle.c: co_legal_moves, co_apply_move; this file is compiled together with it):
 *   in_check(board, side)  = some pseudo-legal move of the other side ends on side's king (false without that king)
 *   strictly legal move    = a pseudo-legal move after which the mover is not in check
 * Every reply is generated and looked at, so nothing here shares logic with the bitboard attack test of cz_rules.cuh.
 * Also the seeded position generators the strict-legality tests use.
 */
#include <stdint.h>
#include <string.h>

int co_legal_moves(const uint8_t *b, int side, uint16_t *out);
int co_apply_move(uint8_t *b, int mv);

int so_in_check(const uint8_t *b, int side) {
    int ksq = -1;
    for (int s = 0; s < 90; s++)
        if (b[s] == (side == 0 ? 1 : 8)) ksq = s;
    if (ksq < 0) return 0;
    uint16_t mv[512];
    const int n = co_legal_moves(b, side ^ 1, mv);
    for (int i = 0; i < n; i++)
        if ((mv[i] >> 7) == ksq) return 1;
    return 0;
}

/* moves: >= 512 entries; legal[i] = 1 iff moves[i] is strictly legal.  Returns the pseudo-legal count. */
int so_strict_moves(const uint8_t *b, int side, uint16_t *moves, uint8_t *legal) {
    const int n = co_legal_moves(b, side, moves);
    for (int i = 0; i < n; i++) {
        uint8_t nb[90];
        memcpy(nb, b, 90);
        co_apply_move(nb, moves[i]);
        legal[i] = (uint8_t)!so_in_check(nb, side);
    }
    return n;
}

/* the output layout of cz_strict_moves_batch */
void so_strict_moves_batch(const uint8_t *boards, const uint8_t *sides, int n, uint16_t *moves /* [n][128] */, int32_t *counts,
                           uint32_t *legal /* [n][4] */, uint8_t *flags) {
    for (int g = 0; g < n; g++) {
        const uint8_t *b = boards + (size_t)g * 90;
        uint16_t mv[512];
        uint8_t ok[512];
        const int c = so_strict_moves(b, sides[g], mv, ok);
        int any = 0;
        counts[g] = c;
        for (int k = 0; k < 4; k++) legal[(size_t)g * 4 + k] = 0;
        for (int i = 0; i < 128; i++) {
            moves[(size_t)g * 128 + i] = i < c ? mv[i] : (uint16_t)0;
            if (i < c && ok[i]) { legal[(size_t)g * 4 + (i >> 5)] |= 1u << (i & 31); any = 1; }
        }
        flags[g] = (uint8_t)((so_in_check(b, sides[g]) ? 1 : 0) | (any ? 0 : 2));
    }
}

static uint64_t rnd(uint64_t *s) { /* splitmix64 */
    uint64_t z = (*s += 0x9E3779B97F4A7C15ull);
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}

static const uint8_t START[90] = {
    3, 5, 4, 2, 1, 2, 4, 5, 3, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 7, 0, 0, 0, 0, 0, 7, 0, 6, 0, 6, 0, 6, 0, 6, 0, 6, 0, 0, 0, 0, 0, 0, 0, 0, 0,
    0, 0, 0, 0, 0, 0, 0, 0, 0, 13, 0, 13, 0, 13, 0, 13, 0, 13, 0, 14, 0, 0, 0, 0, 0, 14, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 10, 12, 11, 9, 8, 9, 11, 12, 10};

/* n positions of uniformly random pseudo-legal play from the start position.  A game goes on until a king is captured (the
 * position after the capture is recorded too), a side has no move, or 400 plies; then the next game starts. */
void so_random_play(uint64_t seed, int n, uint8_t *boards, uint8_t *sides) {
    uint8_t b[90];
    int side = 0, ply = 0;
    memcpy(b, START, 90);
    for (int g = 0; g < n; g++) {
        memcpy(boards + (size_t)g * 90, b, 90);
        sides[g] = (uint8_t)side;
        int hasK = 0, hask = 0;
        for (int s = 0; s < 90; s++) { hasK |= b[s] == 1; hask |= b[s] == 8; }
        uint16_t mv[512];
        const int c = hasK && hask && ply < 400 ? co_legal_moves(b, side, mv) : 0;
        if (c == 0) { memcpy(b, START, 90); side = 0; ply = 0; continue; }
        co_apply_move(b, mv[rnd(&seed) % (uint64_t)c]);
        side ^= 1;
        ply++;
    }
}

/* n set-up boards: every piece of the full set is present with probability `density`/256 and stands on a uniformly random
 * free square -- kings, advisors, bishops and pawns anywhere, so at most one king per colour and sometimes none.  narrow: only
 * files c..g are used, which crowds the palaces so that advisor, bishop and king-step attacks are common. */
void so_random_setup(uint64_t seed, int n, int density, int narrow, uint8_t *boards, uint8_t *sides) {
    static const uint8_t SET[16] = {1, 2, 2, 3, 3, 4, 4, 5, 5, 7, 7, 6, 6, 6, 6, 6};
    for (int g = 0; g < n; g++) {
        uint8_t *b = boards + (size_t)g * 90;
        memset(b, 0, 90);
        for (int colour = 0; colour < 2; colour++)
            for (int i = 0; i < 16; i++) {
                if ((int)(rnd(&seed) & 255) >= density) continue;
                int s;
                do s = narrow ? (int)(rnd(&seed) % 10) * 9 + 2 + (int)(rnd(&seed) % 5) : (int)(rnd(&seed) % 90); while (b[s]);
                b[s] = (uint8_t)(SET[i] + 7 * colour);
            }
        sides[g] = (uint8_t)(rnd(&seed) & 1);
    }
}
