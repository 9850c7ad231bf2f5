// cz_rules.cuh -- warp-cooperative xiangqi rules for sm_90a: bitboard move generation in the
// reference's emission order, move application, flip and the 14-plane encode.
//
// One warp owns one position.  The piece identities sit in a 90-byte mailbox in shared memory (needed for the encode
// and for capture detection); everything the move generator asks about the position -- "is this square empty",
// "is it mine", "where is the first blocker along this rank / file" -- is answered from PACKED BITBOARDS held in
// registers, uniform across the warp (cz::Bits):
//     occ[3], red[3]   90-bit occupancy / red-piece sets, bit s = square s = y*9+x          (rank-major)
//     rocc[3]          the same occupancy in file-major order, bit r = x*10+y                (for vertical rays)
// built with three ballots each from the mailbox (lane l owns squares l, l+32, l+64).  Rook / cannon rays and the
// flying-general test are bit scans (clz / ffs on a 9- or 10-bit line) instead of byte-by-byte walks; knight legs, bishop
// eyes and palace steps are single bit tests.  The side-to-move's pieces (<= 16) are compacted onto lanes 0..15, so the
// critical lane generates ONE piece; an exclusive warp scan over the pieces (= square order) gives the reference's
// y-major / x-minor piece scan with its per-piece direction order (GameBoard.get_legal_moves, main.py:743-1109;
// SURVEY Appendix A.2) byte for byte.
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <stdint.h>

#define CZ_FULL 0xffffffffu
// pure per-lane functions are also compiled for the host so that the CPU test tier can run THIS source against the golden vectors
// (tests/host_rules_harness.cu); the qualifier does not change the device code
#define CZ_HD __host__ __device__ __forceinline__

namespace cz {

// piece kinds after folding colour: 1..7 = K A R B N P C  (pieces_order, main.py:208)
enum { K_ = 1, A_ = 2, R_ = 3, B_ = 4, N_ = 5, P_ = 6, C_ = 7 };

CZ_HD bool piece_red(int p) { return p >= 1 && p <= 7; }
CZ_HD int piece_kind(int p) { return p > 7 ? p - 7 : p; }

// ---- packed position ---------------------------------------------------------------------------------------------
struct Bits {
    uint32_t occ[3], red[3], rocc[3];
};

CZ_HD uint32_t bb_word(const uint32_t (&w)[3], int k) { return k == 0 ? w[0] : k == 1 ? w[1] : w[2]; }
CZ_HD bool bb_test(const uint32_t (&w)[3], int s) { return (bb_word(w, s >> 5) >> (s & 31)) & 1u; }
// `width` (<= 10) bits of a 96-bit set starting at bit `off` (<= 86)
CZ_HD uint32_t bb_line(const uint32_t (&w)[3], int off, int width) {
    const int k = off >> 5, sh = off & 31;
    const uint32_t lo = bb_word(w, k), hi = k >= 2 ? 0u : bb_word(w, k + 1);
    const uint32_t v = sh ? ((lo >> sh) | (hi << (32 - sh))) : lo;
    return v & ((1u << width) - 1u);
}
CZ_HD int bb_msb(uint32_t v) {   // index of the highest set bit, v != 0
#ifdef __CUDA_ARCH__
    return 31 - __clz((int)v);
#else
    return 31 - __builtin_clz(v);
#endif
}
CZ_HD int bb_lsb(uint32_t v) {   // index of the lowest set bit, v != 0
#ifdef __CUDA_ARCH__
    return __ffs((int)v) - 1;
#else
    return __builtin_ctz(v);
#endif
}

// Generates the moves of piece `p` standing on `sq` (it belongs to the side to move) in reference order into out[0..17]
// (a piece has at most 17 moves) and returns the count.  Kings are handled here too (palace steps); the flying-general
// capture is appended by the caller.  No memory is read: every question is a bit test on P.
#define CZ_EMIT(dst) do { out[n] = (uint16_t)(sq | ((dst) << 7)); n++; } while (0)
CZ_HD int gen_piece_bits(const Bits &P, int p, int sq, uint16_t *out) {
    const bool red = piece_red(p);
    const int y = sq / 9, x = sq - y * 9;
    const int kind = piece_kind(p);
    // validate_move (main.py:727-740): the target is empty or holds an enemy  <=>  it does not hold one of mine
    auto mine = [&](int s) { return bb_test(P.occ, s) && (bb_test(P.red, s) == red); };
    auto empty = [&](int s) { return !bb_test(P.occ, s); };
    int n = 0;
    if (kind == R_ || kind == C_) {
        // rays: left (x-1 -> 0), right (x+1 -> 8), towards y-1, towards y+1 (main.py:757-833 / 947-1062)
        const bool cannon = kind == C_;
        const uint32_t rank = bb_line(P.occ, y * 9, 9), file = bb_line(P.rocc, x * 10, 10);
#pragma unroll 1
        for (int d = 0; d < 4; d++) {
            const bool horiz = d < 2, fwd = d & 1;                  // fwd: towards larger coordinate
            const uint32_t line = horiz ? rank : file;
            const int pos = horiz ? x : y, len = horiz ? 9 : 10, step = horiz ? 1 : 9;
            const int base = horiz ? y * 9 : x;                     // square of coordinate 0 on this line
            int first, second = -1;                                 // coordinates of the first / second piece met, or the edge
            if (fwd) {
                uint32_t m = line >> (pos + 1);
                if (m) { first = pos + 1 + bb_lsb(m); m &= m - 1; if (m) second = pos + 1 + bb_lsb(m); }
                else first = len;
                for (int t = pos + 1; t < first; t++) CZ_EMIT(base + t * step);
                if (first < len) {
                    if (!cannon) { if (!mine(base + first * step)) CZ_EMIT(base + first * step); }
                    else if (second >= 0 && !mine(base + second * step)) CZ_EMIT(base + second * step);
                }
            } else {
                uint32_t m = line & ((1u << pos) - 1u);
                if (m) { first = bb_msb(m); m &= ~(1u << first); if (m) second = bb_msb(m); }
                else first = -1;
                for (int t = pos - 1; t > first; t--) CZ_EMIT(base + t * step);
                if (first >= 0) {
                    if (!cannon) { if (!mine(base + first * step)) CZ_EMIT(base + first * step); }
                    else if (second >= 0 && !mine(base + second * step)) CZ_EMIT(base + second * step);
                }
            }
        }
    } else if (kind == N_) {
        // i in (-1,+1), j in (-1,+1): (y+2i, x+j) leg (y+i, x); then (y+i, x+2j) leg (y, x+j)  (835-856)
#pragma unroll
        for (int ij = 0; ij < 4; ij++) {
            const int i = (ij & 2) ? 1 : -1, j = (ij & 1) ? 1 : -1;
            int ty = y + 2 * i, tx = x + j;
            if (ty >= 0 && ty < 10 && tx >= 0 && tx < 9 && !mine(ty * 9 + tx) && empty((y + i) * 9 + x)) CZ_EMIT(ty * 9 + tx);
            ty = y + i; tx = x + 2 * j;
            if (ty >= 0 && ty < 10 && tx >= 0 && tx < 9 && !mine(ty * 9 + tx) && empty(y * 9 + x + j)) CZ_EMIT(ty * 9 + tx);
        }
    } else if (kind == B_) {
        // i in (-2,+2): (y+i, x+i) then (y+i, x-i); own half only; eye must be empty (857-888)
#pragma unroll
        for (int i = -2; i <= 2; i += 4) {
            const int h = i / 2, ty = y + i;
            if (ty < 0 || ty > 9 || (red ? ty > 4 : ty < 5)) continue;
            int tx = x + i;
            if (tx >= 0 && tx < 9 && !mine(ty * 9 + tx) && empty((y + h) * 9 + x + h)) CZ_EMIT(ty * 9 + tx);
            tx = x - i;
            if (tx >= 0 && tx < 9 && !mine(ty * 9 + tx) && empty((y + h) * 9 + x - h)) CZ_EMIT(ty * 9 + tx);
        }
    } else if (kind == A_) {
        // i in (-1,+1): (y+i, x+i) then (y+i, x-i); palace only (889-918)
#pragma unroll
        for (int i = -1; i <= 1; i += 2) {
            const int ty = y + i;
            if (ty < 0 || ty > 9 || (red ? ty > 2 : ty < 7)) continue;
            int tx = x + i;
            if (tx >= 3 && tx <= 5 && !mine(ty * 9 + tx)) CZ_EMIT(ty * 9 + tx);
            tx = x - i;
            if (tx >= 3 && tx <= 5 && !mine(ty * 9 + tx)) CZ_EMIT(ty * 9 + tx);
        }
    } else if (kind == K_) {
        // (y, x-1), (y, x+1), (y-1, x), (y+1, x) inside the own palace (919-946)
#pragma unroll
        for (int k = 0; k < 4; k++) {
            const int ty = y + (k == 2 ? -1 : k == 3 ? 1 : 0), tx = x + (k == 0 ? -1 : k == 1 ? 1 : 0);
            if (ty < 0 || ty > 9 || tx < 3 || tx > 5 || (red ? ty > 2 : ty < 7)) continue;
            if (!mine(ty * 9 + tx)) CZ_EMIT(ty * 9 + tx);
        }
    } else {  // P_
        // forward (red y+1 / black y-1); after the river x+1 then x-1 (1063-1095)
        const int ty = red ? y + 1 : y - 1;
        if (ty >= 0 && ty < 10 && !mine(ty * 9 + x)) CZ_EMIT(ty * 9 + x);
        if (red ? y > 4 : y < 5) {
            if (x < 8 && !mine(sq + 1)) CZ_EMIT(sq + 1);
            if (x > 0 && !mine(sq - 1)) CZ_EMIT(sq - 1);
        }
    }
    return n;
}
#undef CZ_EMIT

// flying general (main.py:1097-1107): both kings on one file and no piece on the rows K_y < i < k_y.  (The reference's
// range(K_y + 1, k_y) is empty when the red king stands above the black one -- impossible in play, kept for exactness.)
CZ_HD bool kings_face(const Bits &P, int Ksq, int ksq) {
    if (Ksq < 0 || ksq < 0 || (Ksq % 9) != (ksq % 9)) return false;
    const int x = Ksq % 9, yK = Ksq / 9, yk = ksq / 9;
    const uint32_t file = bb_line(P.rocc, x * 10, 10);
    const uint32_t between = yk > yK ? (((1u << yk) - 1u) & ~((2u << yK) - 1u)) : 0u;
    return (file & between) == 0;
}

// serial construction of the bitboards (host harness; the device builds them with ballots, see warp_bits)
CZ_HD void bits_from_board(const uint8_t *b, Bits &P) {
    for (int k = 0; k < 3; k++) P.occ[k] = P.red[k] = P.rocc[k] = 0;
    for (int s = 0; s < 90; s++) {
        const int p = b[s];
        if (!p) continue;
        const int y = s / 9, x = s - y * 9, r = x * 10 + y;
        P.occ[s >> 5] |= 1u << (s & 31);
        if (piece_red(p)) P.red[s >> 5] |= 1u << (s & 31);
        P.rocc[r >> 5] |= 1u << (r & 31);
    }
}

// ---- strict legality ---------------------------------------------------------------------------------------------
// in_check(board, side): some pseudo-legal move of the OTHER side, as gen_piece_bits / kings_face list them, ends on the
// square of `side`'s king (false when that king is absent).  A pseudo-legal move is strictly legal iff the mover is not in
// check after it.  No replies are generated: `attacked` asks, from the king's square, where each kind of attacker would
// have to stand, with the attacker's own placement rules exactly as gen_piece_bits applies them to its targets.

// The position after moving src -> dst, never materialised: the bitboards are patched in registers and a piece is looked up
// as "dst holds what stood on src, src is empty, everything else is the board b".  src = dst = -1 is the board itself.
struct Moved {
    const uint8_t *b;
    int src, dst;
    CZ_HD int at(int s) const { return s == dst ? b[src] : s == src ? 0 : b[s]; }
};

CZ_HD void bb_put(uint32_t (&w)[3], int s, bool v) {
#pragma unroll
    for (int k = 0; k < 3; k++) {
        const uint32_t m = (s >> 5) == k ? 1u << (s & 31) : 0u;
        w[k] = v ? (w[k] | m) : (w[k] & ~m);
    }
}

// P after the piece on src (of colour mover_red) moved to dst; a capture needs no extra step
CZ_HD Bits bits_after(const Bits &P, int src, int dst, bool mover_red) {
    Bits Q = P;
    bb_put(Q.occ, src, false); bb_put(Q.red, src, false); bb_put(Q.rocc, (src % 9) * 10 + src / 9, false);
    bb_put(Q.occ, dst, true); bb_put(Q.red, dst, mover_red); bb_put(Q.rocc, (dst % 9) * 10 + dst / 9, true);
    return Q;
}

// Is the king of `side` on ksq attacked in the position (P, M)?  esq: the other king's square or -1.
CZ_HD bool attacked(const Bits &P, const Moved &M, int side, int ksq, int esq) {
    const int foe = side == 0 ? 7 : 0;                  // piece code of an attacker of kind k is k + foe
    const bool foe_red = side != 0;
    const int y = ksq / 9, x = ksq - y * 9;
    // rook = first piece met along the rank / file, cannon = second
    const uint32_t rank = bb_line(P.occ, y * 9, 9), file = bb_line(P.rocc, x * 10, 10);
#pragma unroll 1
    for (int d = 0; d < 4; d++) {
        const bool horiz = d < 2, fwd = d & 1;
        const uint32_t line = horiz ? rank : file;
        const int pos = horiz ? x : y, step = horiz ? 1 : 9, base = horiz ? y * 9 : x;
        int first = -1, second = -1;
        if (fwd) {
            uint32_t m = line >> (pos + 1);
            if (m) { first = pos + 1 + bb_lsb(m); m &= m - 1; if (m) second = pos + 1 + bb_lsb(m); }
        } else {
            uint32_t m = line & ((1u << pos) - 1u);
            if (m) { first = bb_msb(m); m &= ~(1u << first); if (m) second = bb_msb(m); }
        }
        if (first >= 0 && M.at(base + first * step) == R_ + foe) return true;
        if (second >= 0 && M.at(base + second * step) == C_ + foe) return true;
    }
    // knight: both knight squares beyond a diagonal neighbour share it as their leg (the square next to the knight)
#pragma unroll
    for (int ij = 0; ij < 4; ij++) {
        const int i = (ij & 2) ? 1 : -1, j = (ij & 1) ? 1 : -1;
        const int ly = y + i, lx = x + j;
        if (ly < 0 || ly > 9 || lx < 0 || lx > 8 || bb_test(P.occ, ly * 9 + lx)) continue;
        if (y + 2 * i >= 0 && y + 2 * i <= 9 && M.at((y + 2 * i) * 9 + lx) == N_ + foe) return true;
        if (x + 2 * j >= 0 && x + 2 * j <= 8 && M.at(ly * 9 + x + 2 * j) == N_ + foe) return true;
    }
    // pawn: from behind (its forward step), and from either side once it stands beyond its river
    {
        const int py = foe_red ? y - 1 : y + 1;
        if (py >= 0 && py <= 9 && M.at(py * 9 + x) == P_ + foe) return true;
        if (foe_red ? y > 4 : y < 5) {
            if (x > 0 && M.at(ksq - 1) == P_ + foe) return true;
            if (x < 8 && M.at(ksq + 1) == P_ + foe) return true;
        }
    }
    // bishop: two diagonal steps with an empty eye; it only lands in its own half
    if (foe_red ? y <= 4 : y >= 5) {
#pragma unroll
        for (int ij = 0; ij < 4; ij++) {
            const int i = (ij & 2) ? 1 : -1, j = (ij & 1) ? 1 : -1;
            const int by = y + 2 * i, bx = x + 2 * j;
            if (by < 0 || by > 9 || bx < 0 || bx > 8) continue;
            if (!bb_test(P.occ, (y + i) * 9 + x + j) && M.at(by * 9 + bx) == B_ + foe) return true;
        }
    }
    // advisor and the king's palace step: they only land inside their own palace
    if (x >= 3 && x <= 5 && (foe_red ? y <= 2 : y >= 7)) {
#pragma unroll
        for (int ij = 0; ij < 4; ij++) {
            const int ay = y + ((ij & 2) ? 1 : -1), ax = x + ((ij & 1) ? 1 : -1);
            if (ay >= 0 && ay <= 9 && ax >= 0 && ax <= 8 && M.at(ay * 9 + ax) == A_ + foe) return true;
        }
        if (esq >= 0) {
            const int ey = esq / 9, ex = esq - ey * 9;
            if ((ey == y && (ex == x - 1 || ex == x + 1)) || (ex == x && (ey == y - 1 || ey == y + 1))) return true;
        }
    }
    // flying general, the same test that appends the capture to the move list
    return side == 0 ? kings_face(P, ksq, esq) : kings_face(P, esq, ksq);
}

// in_check of the board itself.  Ksq / ksq: the king squares (-1 if absent).
CZ_HD bool in_check(const Bits &P, const uint8_t *b, int side, int Ksq, int ksq) {
    const int mine = side == 0 ? Ksq : ksq, other = side == 0 ? ksq : Ksq;
    return mine >= 0 && attacked(P, Moved{b, -1, -1}, side, mine, other);
}

// Is the pseudo-legal move mv of `side` strictly legal on (P, b)?
CZ_HD bool move_is_strict(const Bits &P, const uint8_t *b, int side, int mv, int Ksq, int ksq) {
    const int src = mv & 127, dst = (mv >> 7) & 127;
    int mine = side == 0 ? Ksq : ksq, other = side == 0 ? ksq : Ksq;
    if (src == mine) mine = dst;                        // the king itself moves
    if (dst == other) other = -1;                       // the other king is captured
    if (mine < 0) return true;
    return !attacked(bits_after(P, src, dst, side == 0), Moved{b, src, dst}, side, mine, other);
}

#ifdef __CUDACC__
__device__ __forceinline__ int warp_excl_scan(int v, int lane, int &total) {
    int inc = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        int t = __shfl_up_sync(CZ_FULL, inc, o);
        if (lane >= o) inc += t;
    }
    total = __shfl_sync(CZ_FULL, inc, 31);
    return inc - v;
}

// Per-warp scratch of the move generator: the squares of the mover's pieces and one 18-entry slot per lane.
struct MoveScratch {
    uint16_t slot[32 * 18];
    uint8_t sq[96];
};

// Bitboards of the position in the warp's mailbox b (shared memory, 90 bytes + 6 pad).  Also returns the king squares (-1 if absent).
__device__ __forceinline__ void warp_bits(const uint8_t *b, int lane, Bits &P, int &Ksq, int &ksq) {
    Ksq = ksq = -1;
#pragma unroll
    for (int k = 0; k < 3; k++) {
        const int s = lane + 32 * k;
        const int p = s < 90 ? b[s] : 0;
        int q = 0;
        if (s < 90) { const int x = s / 10, y = s - x * 10; q = b[y * 9 + x]; }     // file-major bit s = square (x, y)
        P.occ[k] = __ballot_sync(CZ_FULL, p != 0);
        P.red[k] = __ballot_sync(CZ_FULL, p >= 1 && p <= 7);
        P.rocc[k] = __ballot_sync(CZ_FULL, q != 0);
        const unsigned Km = __ballot_sync(CZ_FULL, p == 1), km = __ballot_sync(CZ_FULL, p == 8);
        if (Km) Ksq = 32 * k + __ffs(Km) - 1;      // at most one king of each colour
        if (km) ksq = 32 * k + __ffs(km) - 1;
    }
}

// Warp-cooperative GameBoard.get_legal_moves.  b: 90-byte board in shared memory, moves: shared uint16[>=136].
// Returns the move count (uniform across the warp).  All 32 lanes must call, converged.
__device__ __noinline__ int warp_legal_moves(const uint8_t *b, int side, uint16_t *moves, MoveScratch &T, int lane) {
    Bits P;
    int Ksq, ksq;
    warp_bits(b, lane, P, Ksq, ksq);
    // list the mover's pieces in square order: piece r stands on T.sq[r]
    int np = 0;
#pragma unroll
    for (int k = 0; k < 3; k++) {
        const uint32_t own = side == 0 ? P.red[k] : (P.occ[k] & ~P.red[k]);
        if ((own >> lane) & 1u) T.sq[np + __popc(own & ((1u << lane) - 1u))] = (uint8_t)(lane + 32 * k);
        np += __popc(own);
    }
    __syncwarp();
    // one piece per lane (a side has <= 16 pieces in play: a single pass; arbitrary set-up positions take more)
    int n = 0;
    for (int base = 0; base < np; base += 32) {
        int c = 0;
        if (base + lane < np) {
            const int sq = T.sq[base + lane];
            c = gen_piece_bits(P, b[sq], sq, T.slot + lane * 18);
        }
        int tot;
        const int off = n + warp_excl_scan(c, lane, tot);      // exclusive scan over the pieces = the reference's square scan
        for (int j = 0; j < c; j++)
            if (off + j < 136) moves[off + j] = T.slot[lane * 18 + j];
        n += tot;
        __syncwarp();
    }
    // flying general: the mover's king takes, appended LAST (1097-1107)
    if (kings_face(P, Ksq, ksq)) {
        if (lane == 0 && n < 136) moves[n] = side == 0 ? (uint16_t)(Ksq | (ksq << 7)) : (uint16_t)(ksq | (Ksq << 7));
        n++;
    }
    __syncwarp();
    return n;
}

// warp_legal_moves (same list, order and count) plus strict legality: bit i of the 128-bit legal mask is set iff move i
// leaves the mover's king unattacked (bits at and above min(count, 128) are zero); flags bit 0 = the mover is in check,
// bit 1 = mated (no strictly legal move: checkmate or stalemate).  Lane l tests moves l, l + 32, l + 64, l + 96, each
// against bitboards patched in its own registers; nothing but the mailbox b is read.  All 32 lanes must call, converged.
__device__ __forceinline__ int warp_strict_moves(const uint8_t *b, int side, uint16_t *moves, MoveScratch &T, int lane,
                                                 uint32_t (&legal)[4], int &flags) {
    const int n = warp_legal_moves(b, side, moves, T, lane);
    Bits P;
    int Ksq, ksq;
    warp_bits(b, lane, P, Ksq, ksq);
    uint32_t any = 0;
#pragma unroll
    for (int k = 0; k < 4; k++) {
        const int i = lane + 32 * k;
        const bool ok = i < n && move_is_strict(P, b, side, moves[i], Ksq, ksq);
        legal[k] = __ballot_sync(CZ_FULL, ok);
        any |= legal[k];
    }
    flags = (in_check(P, b, side, Ksq, ksq) ? 1 : 0) | (any ? 0 : 2);
    return n;
}
#endif  // __CUDACC__

// swap colour of a piece code (try_flip's swapcase, main.py:566-572)
CZ_HD int swap_colour(int p) { return p == 0 ? 0 : (p <= 7 ? p + 7 : p - 7); }

template <typename T> CZ_HD T enc_one();
template <> CZ_HD float enc_one<float>() { return 1.0f; }
template <> CZ_HD __nv_bfloat16 enc_one<__nv_bfloat16>() { return __float2bfloat16(1.0f); }
template <> CZ_HD __half enc_one<__half>() { return __float2half(1.0f); }

// Warp-cooperative generate_inputs (main.py:531-557): flip for black (rows reversed, colours
// swapped), then T[rank][file][plane] for rank < 9, file < 10 reads board cell rank*9+file --
// the reference's indexing, which drops squares 82..89 and reads 8 cells twice (SURVEY 0.5).
// out: 1260 elements of T in global memory (row of the NN batch), 16-byte aligned.
template <typename T>
__host__ __device__ void warp_encode(const uint8_t *b, int side, T *out, int lane) {
    constexpr int VEC = 16 / sizeof(T);           // elements per 16-byte store
    constexpr int NV = 1260 / VEC;                // 315 (f32) or 157.5 -> handled below
    static_assert(1260 % (VEC / 2) == 0, "row must be a multiple of 8 bytes");
    if constexpr (sizeof(T) == 4) {
        for (int v = lane; v < NV; v += 32) {
            float4 o;
            float *of = reinterpret_cast<float *>(&o);
#pragma unroll
            for (int e = 0; e < 4; e++) {
                const int k = v * 4 + e, cell = k / 14, plane = k - cell * 14;
                const int rank = cell / 10, file = cell - rank * 10, s = rank * 9 + file;
                int p;
                if (side == 0) p = b[s];
                else { const int yy = s / 9, xx = s - yy * 9; p = swap_colour(b[(9 - yy) * 9 + xx]); }
                of[e] = (p - 1 == plane) ? 1.0f : 0.0f;
            }
            reinterpret_cast<float4 *>(out)[v] = o;
        }
    } else {
        // 2-byte element types: 1260 * 2 = 2520 B = 315 8-byte stores
        for (int v = lane; v < 315; v += 32) {
            T o[4];
#pragma unroll
            for (int e = 0; e < 4; e++) {
                const int k = v * 4 + e, cell = k / 14, plane = k - cell * 14;
                const int rank = cell / 10, file = cell - rank * 10, s = rank * 9 + file;
                int p;
                if (side == 0) p = b[s];
                else { const int yy = s / 9, xx = s - yy * 9; p = swap_colour(b[(9 - yy) * 9 + xx]); }
                o[e] = (p - 1 == plane) ? enc_one<T>() : T(0.0f);
            }
            reinterpret_cast<uint2 *>(out)[v] = *reinterpret_cast<uint2 *>(o);
        }
    }
}

}  // namespace cz
