// TEST INFRASTRUCTURE.  The strict-legality functions of cchess_zero_b200/csrc/cz_rules.cuh (attacked / in_check / move_is_strict)
// compiled FOR THE HOST, with cz::warp_strict_moves' warp plumbing replaced by its serial meaning: the move list is
// hr_legal_moves', lane l of ballot k tests move l + 32 k.  Output layout = k_strict_moves'.
#include "host_rules_harness.cu"

extern "C" int hr_strict_moves(const uint8_t *board, int side, uint16_t *out /* >= 256 */, uint32_t *legal /* [4] */, int *flags) {
    const int n = hr_legal_moves(board, side, out);
    cz::Bits P;
    cz::bits_from_board(board, P);
    int Ksq = -1, ksq = -1;
    for (int sq = 0; sq < 90; sq++) {
        if (board[sq] == 1) Ksq = sq;
        if (board[sq] == 8) ksq = sq;
    }
    uint32_t any = 0;
    for (int k = 0; k < 4; k++) {
        legal[k] = 0;
        for (int lane = 0; lane < 32; lane++) {
            const int i = lane + 32 * k;
            if (i < n && cz::move_is_strict(P, board, side, out[i], Ksq, ksq)) legal[k] |= 1u << lane;
        }
        any |= legal[k];
    }
    *flags = (cz::in_check(P, board, side, Ksq, ksq) ? 1 : 0) | (any ? 0 : 2);
    return n;
}

extern "C" void hr_strict_moves_batch(const uint8_t *boards, const uint8_t *sides, int n, uint16_t *moves /* [n][128] */, int32_t *counts,
                                      uint32_t *legal /* [n][4] */, uint8_t *flags) {
    for (int g = 0; g < n; g++) {
        uint16_t out[256];
        int fl;
        const int c = hr_strict_moves(boards + (size_t)g * 90, sides[g], out, legal + (size_t)g * 4, &fl);
        counts[g] = c;
        flags[g] = (uint8_t)fl;
        for (int i = 0; i < 128; i++) moves[(size_t)g * 128 + i] = i < c ? out[i] : (uint16_t)0;
    }
}
