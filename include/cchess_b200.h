/*
 * cchess_b200.h -- C ABI of the batched MCTS self-play engine (H100, sm_90a).
 *
 * The reference (chengstone/cchess-zero) is pure Python and has no FFI; this header is
 * the boundary a maintainer would bind from the reference's Python (ctypes stub in
 * INTEGRATION.md).  Each entry point names the reference code it replaces
 * (file:line relative to the reference tree).
 *
 * Conventions
 *   - every function returns an int status: CZ_OK (0) or a negative CZ_E* code; nothing
 *     throws across the boundary; cz_last_error() gives a thread-local message.
 *   - plain pointers and sizes only.  "host" buffers are ordinary (ideally pinned) host
 *     memory owned by the caller; "dev" pointers are CUDA device pointers owned by the
 *     caller (e.g. torch tensors' data_ptr()).  `stream` is a cudaStream_t passed as void*
 *     (NULL = default stream); asynchronous work is ordered on it.
 *   - boards are 90 bytes, row-major sq = y*9 + x (y = rank 0..9 = row of the reference's
 *     state string, x = file a..i), piece codes 0 = empty, 1..7 = K A R B N P C (red /
 *     upper-case / 'w'), 8..14 = k a r b n p c (black / 'b')  [pieces_order, main.py:208].
 *   - a move is uint16: src_sq | dst_sq << 7.   side: 0 = 'w' (red), 1 = 'b'.
 *   - a handle is bound to one GPU; calls on one handle are not thread-safe.
 */
#ifndef CCHESS_B200_H
#define CCHESS_B200_H
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define CZ_OK 0
#define CZ_EINVAL (-1)   /* bad argument */
#define CZ_ECUDA (-2)    /* CUDA runtime error (see cz_last_error) */
#define CZ_ENOMEM (-3)   /* allocation failed */
#define CZ_EENGINE (-4)  /* a game raised an engine error flag (see cz_engine_counters) */

#define CZ_NSQ 90
#define CZ_NLABEL 2086       /* labels_len, main.py:212 */
#define CZ_MAXCHILD 128      /* upper bound on pseudo-legal moves of one position */
#define CZ_ENC_LEN 1260      /* 9*10*14, main.py:550 */

/* nn input element types accepted by encode / wave */
#define CZ_F32 0
#define CZ_BF16 1
#define CZ_F16 2
#define CZ_BOARD 3           /* wave only: row g = 96 bytes, the side-to-move-canonical board (for cz_net_first_conv) */

/* per-game error flags (cz_engine_counters) */
#define CZ_ERR_NOMOVES 1     /* expanded node with zero legal moves (reference: ValueError from max(), main.py:159) */
#define CZ_ERR_NOLABEL 2     /* move outside the 2086-label table (reference: KeyError, main.py:181) */
#define CZ_ERR_DEPTH 4       /* search path deeper than the path stack */
#define CZ_ERR_ARENA 8       /* tree arena exhausted */
#define CZ_ERR_CHILDREN 16   /* more than CZ_MAXCHILD moves */
#define CZ_ERR_ILLEGAL 32    /* cz_engine_play_moves: move not legal at the game's root (game left unchanged) */

const char *cz_last_error(void);
int cz_version(void);

/* ---- move-label codec: create_uci_labels main.py:30-65, label2i 217, unflipped_index 213-214 ---- */
int cz_labels(char *out /* [2086*4] host, no terminators */);
int cz_label_index(int src_sq, int dst_sq);           /* >= 0 label index, -1 if not a label */
int cz_unflipped_index(int32_t *out /* [2086] host */);

/* ---- state strings: GameBoard.board_to_pos_name main.py:705-714, re-compression 691-699 ---- */
int cz_from_state(const char *state, uint8_t *board /* [90] */);
int cz_to_state(const uint8_t *board, char *out /* >= 100 bytes */);

/* ---- stateless, batched rules; HOST buffers, computed on the GPU (copies included) ----
 * cz_legal_moves_batch  replaces GameBoard.get_legal_moves            main.py:743-1109 (same ORDER)
 * cz_apply_moves_batch  replaces GameBoard.sim_do_action + is_kill_move  main.py:647-702, 219-227
 * cz_encode_batch       replaces MCTS_tree.generate_inputs (try_flip + state_to_positions, incl. the
 *                       rank*9+file indexing of the [9][10][14] tensor) main.py:531-574            */
int cz_legal_moves_batch(int device, const uint8_t *boards /* [n][90] */, const uint8_t *sides /* [n] */, int n,
                         uint16_t *moves /* [n][128] */, int32_t *counts /* [n] */);
int cz_apply_moves_batch(int device, uint8_t *boards /* [n][90] in/out */, const uint16_t *moves /* [n] */, int n,
                         uint8_t *captured /* [n] piece code captured or 0 */);
int cz_encode_batch(int device, const uint8_t *boards, const uint8_t *sides, int n, float *out /* [n][9][10][14] */);
/* device-pointer variants (no copies; async on stream) */
int cz_legal_moves_dev(const uint8_t *boards, const uint8_t *sides, int n, uint16_t *moves, int32_t *counts, void *stream);
int cz_encode_dev(const uint8_t *boards, const uint8_t *sides, int n, void *out, int dtype, void *stream);

/* ---- strict legality (no counterpart in the reference, whose moves are pseudo-legal and whose games end by king capture) ----
 * in_check(board, side): some pseudo-legal move of the other side, flying general included, ends on side's king (false when
 * that king is absent).  A pseudo-legal move is strictly legal iff the mover is not in check after it; a side without a
 * strictly legal move is mated (checkmate or stalemate, both lose).  Boards may be any placement with at most one king per colour.
 * Per position:  moves / counts  exactly what cz_legal_moves_batch writes for the same input (a count above CZ_MAXCHILD is
 *                                returned as it is and the list is truncated);
 *                legal u32[4]    bit i & 31 of word i >> 5 is set iff move i is strictly legal; bits at and above
 *                                min(count, 128) are zero;
 *                flags u8        bit 0 (CZ_IN_CHECK) = in_check(board, side), bit 1 (CZ_MATED) = no strictly legal move.
 * The batch form takes host buffers (null / n < 0 -> CZ_EINVAL, n == 0 -> CZ_OK); the dev form takes device pointers, launches
 * on `stream`, and neither allocates nor synchronises. */
#define CZ_IN_CHECK 1
#define CZ_MATED 2
int cz_strict_moves_batch(int device, const uint8_t *boards /* [n][90] */, const uint8_t *sides /* [n] */, int n,
                          uint16_t *moves /* [n][128] */, int32_t *counts /* [n] */, uint32_t *legal /* [n][4] */, uint8_t *flags /* [n] */);
int cz_strict_moves_dev(const uint8_t *boards, const uint8_t *sides, int n, uint16_t *moves, int32_t *counts, uint32_t *legal,
                        uint8_t *flags, void *stream);

/* ---- replay buffer -> training mini-batch (cchess_main.policy_update's data path, main.py:1160-1166 + run() 1236-1239) ----
 * The ring holds cap records in device arrays: boards u8 [cap][90] (side-to-move canonical), n u8 [cap], idx i16 [cap][128]
 * (label indices), prob f32 [cap][128] (visit probabilities), z f32 [cap].  Output row r is ring record rows[r]:
 *   planes f32 [m][9][10][14]  = MCTS_tree.state_to_positions(state) (main.py:547-557, incl. its rank*9+file indexing)
 *   pi     f32 [m][2086]       = the dense pi vector: zeros, prob[k] at label idx[k] for k < n
 *   zout   f32 [m]             = z
 * mirror (dev u8 [m] or NULL): rows with mirror[r] != 0 are mirrored left to right (file x -> 8 - x) -- the board before it
 * is encoded, each probability to the mirrored move's label (cz_mirror_labels).  rows, mirror and all arrays are DEVICE
 * pointers; planes 16-byte, pi 8-byte aligned.  Asynchronous on `stream`, no allocation: capturable in a CUDA graph -- except
 * the first call with a mirror array on a device, which uploads the 4 KB mirror table (synchronous; m may be 0 for that).
 * Row indices and record contents (n <= 128, 0 <= idx < 2086) are the caller's to validate; invalid ones are skipped.
 * CZ_EINVAL: m < 0, cap < 0, a NULL array with m > 0, cap == 0 with m > 0, misaligned outputs. */
int cz_replay_batch(const uint8_t *boards, const uint8_t *n, const int16_t *idx, const float *prob, const float *z, int cap,
                    const int32_t *rows, const uint8_t *mirror, int m, float *planes, float *pi, float *zout, void *stream);
/* The left-right mirror of every label: out[i] = label of label i with both files x -> 8 - x (host [2086]).  The table is
 * closed under the mirror and an involution (checked when the label table is built; CZ_EINVAL otherwise). */
int cz_mirror_labels(int16_t *out /* [2086] host */);

/* ---- the batched engine: n_games independent (GameBoard, MCTS_tree) pairs resident in HBM ---- */
typedef struct cz_engine cz_engine;

/* arena_words: uint32 words of tree storage per game per half (two halves, ping-pong re-rooting);
 * 0 selects the default (2 Mi words = 8 MiB per half; a 1200-playout self-play soak peaks at 0.74 Mi words). */
int cz_engine_create(int n_games, int64_t arena_words, int device, cz_engine **out);
/* Leaf-parallel variant: up to `leaves` (1..64) leaves per game per wave inside one tree (virtual-loss batching; the
 * search_threads > 1 idea of main.py:337-440 with a deterministic schedule of its own -- not bit-comparable with the
 * reference's coroutine interleaving).  Network rows are then g*leaves + slot: nn_in [n_games*leaves][...],
 * logits [n_games*leaves][2086], value [n_games*leaves].  leaves == 1 is cz_engine_create; leaves == -1 runs the
 * leaf-parallel kernel with a single slot (test hook: must equal the one-leaf kernel bit for bit). */
int cz_engine_create_ex(int n_games, int64_t arena_words, int device, int leaves, cz_engine **out);
/* search_threads = K > 1 EXACTLY as the reference schedules it (main.py:337-470 on uvloop), in canonical deterministic form: every
 * playout is a task, at most K hold the semaphore, the event loop's FIFO batches, the two-hop asyncio.sleep(1e-4) spin on
 * now_expanding nodes and prediction_worker's batching are simulated per game by one warp (k_wave_fifo); node blocks carry the
 * stored Q of back_up_value (main.py:193) because concurrent virtual losses make it differ from W/N.  Specification:
 * oracle/detloop.py (the reference's own coroutines on a deterministic loop) and the C oracle (co_tree_search_fifo), both
 * pinned to real uvloop runs of the reference (tests/golden/k16_stats.json.gz).  Network rows as for `leaves`: g*K + slot.
 * search_threads: 1..32 (1 reproduces cz_engine_create's results with the 6-array blocks). */
int cz_engine_create_fifo(int n_games, int64_t arena_words, int device, int search_threads, cz_engine **out);
int cz_engine_is_fifo(const cz_engine *e);
int cz_engine_leaves(const cz_engine *e);
/* A one-leaf engine (cz_engine_create) that plays by the given rules.
 *   CZ_RULES_REFERENCE: the reference's rules (pseudo-legal moves; a game ends when a king is taken): cz_engine_create's engine.
 *   CZ_RULES_STRICT:    the full rules of xiangqi.  A node's children are its strictly legal moves (the subset of the pseudo-legal
 *                       list that leaves the mover's king unattacked, cz_strict_moves_batch, in the same order; priors normalised over
 *                       them).  A node without one is mated (checkmate and stalemate both lose): it is expanded with no children, the
 *                       playout that expanded it backs up as if the network had returned -1 for the side to move there, and later
 *                       descents onto it end there worth +1 to the move into it.  A root without a strictly legal move ends the game
 *                       with terminal code 3 after cz_engine_reset / set_root_meta / play / play_moves (one extra kernel launch each);
 *                       cz_engine_play_moves on an unexpanded root accepts only strictly legal moves among the first 128 pseudo-legal
 *                       ones (the moves an expansion keeps; more than 128 is CZ_ERR_CHILDREN, possible on set-up boards only).  A king capture stays legal and
 *                       terminal (set-up positions only).  Snapshots are written in format 2.
 * Any other value: CZ_EINVAL.  Leaf-parallel and search_threads = K engines play by the reference rules only. */
#define CZ_RULES_REFERENCE 0
#define CZ_RULES_STRICT 1
int cz_engine_create_rules(int n_games, int64_t arena_words, int device, int rules, cz_engine **out);
int cz_engine_rules(const cz_engine *e);
/* How an expansion turns the leaf's logits l_i (its children's label entries, in move order) into priors; any engine kind.
 *   CZ_PRIORS_REFERENCE: P_i = l_i / (1e-8 + the serial f32 sum of the l_i), the reference's leaf_node.expand (the default).
 *   CZ_PRIORS_SOFTMAX:   P_i = f32(e_i / s), e_i = exp(f64(l_i) - f64(m)) with m the largest l_i (NaNs ignored, as fmaxf) and
 *                        s the f64 sum of the e_i in move order; exp is the library's own (csrc/cz_exp.h; DESIGN 3k).
 * cz_engine_set_priors: CZ_EINVAL for another mode, and for any call once the engine has run a wave (so that a captured graph never
 * holds the other kernel instantiation); the engine is unchanged then.  cz_engine_priors: the mode, or CZ_EINVAL for a null engine. */
#define CZ_PRIORS_REFERENCE 0
#define CZ_PRIORS_SOFTMAX 1
int cz_engine_set_priors(cz_engine *e, int mode);
int cz_engine_priors(const cz_engine *e);
int cz_engine_destroy(cz_engine *e);
int cz_engine_n_games(const cz_engine *e);

/* GameBoard.reload (main.py:604-608) + MCTS_tree.reload (255-258) for the games with mask[g] != 0
 * (mask NULL = all).  boards/sides/rr NULL = the start position, 'w', 0. All host pointers. */
int cz_engine_reset(cz_engine *e, void *stream, const uint8_t *mask, const uint8_t *boards, const uint8_t *sides,
                    const int32_t *rr);

/* Override side-to-move / restrict_round of the root without touching the tree: MCTS_tree.main takes
 * current_player and restrict_round as call arguments (main.py:473).  Host pointers, any may be NULL. */
int cz_engine_set_root_meta(cz_engine *e, void *stream, const uint8_t *mask, const uint8_t *sides, const int32_t *rr);

/* Start a search of `playouts` playouts (MCTS_tree.main's loop count, main.py:490) on the games with
 * mask[g] != 0 (NULL = every non-terminal game). */
int cz_engine_begin_search(cz_engine *e, void *stream, const uint8_t *mask, int playouts);

/* One wave = one kernel launch (capturable in a CUDA graph; no host sync, no allocation):
 *   1. for every game with a pending leaf: expand it from logits/value of the previous wave
 *      (leaf_node.expand main.py:175-187 incl. flip_policy 1152-1155 and the legal-move generation),
 *      undo the virtual loss and back the value up (main.py:426-435, 189-194);
 *   2. run playouts of start_tree_search (main.py:350-440, search_threads = 1 semantics) until the
 *      game needs a network evaluation: PUCT selection (108-116, 158-159), virtual loss (403-404),
 *      terminal / 60-ply rule (409-416); terminal playouts are backed up in-kernel and the game
 *      continues with its next playout;
 *   3. encode the leaf (main.py:531-557) into row g of nn_in.
 * nn_in: dev [n_games][9][10][14] of `nn_dtype`; logits: dev f32 [n_games][2086]; value: dev f32 [n_games].
 * A game's row of logits/value is only read if that game has a pending leaf.                              */
int cz_engine_wave(cz_engine *e, void *stream, void *nn_in, int nn_dtype, const float *logits, const float *value);
/* search_threads = K engines (cz_engine_create_fifo): one wave WITH ROW COMPACTION of the K-rows-per-game network batch.  On average
 * ~11 of the 16 slots of a searching game carry a leaf (the rest spin on a node that is being expanded, main.py:354-355), and games
 * whose search is complete carry none; evaluating only those rows is what the reference's prediction_worker does (main.py:442-464
 * evaluates "whatever is queued").  nn_stage [B*K rows] is written like cz_engine_wave's nn_in; nn_dense [B*K rows] receives the rows
 * that need an evaluation, densely, in (game, slot) order; logits / value are read through the row map of the PREVIOUS call: between
 * two calls the caller evaluates nn_dense[0 .. n) into logits[0 .. n) / value[0 .. n), n = cz_engine_live_rows (stream sync).
 * Results are identical to cz_engine_wave's whenever the evaluator is row-independent. */
int cz_engine_wave_compact(cz_engine *e, void *stream, void *nn_stage, void *nn_dense, int nn_dtype, const float *logits, const float *value);
int cz_engine_live_rows(cz_engine *e, void *stream, int32_t *out_rows);

/* Board hashing (north_star): when switched on, every wave also leaves the 64-bit Zobrist key of each pending leaf's position
 * (piece-square keys XOR side-to-move key, maintained incrementally along the descent; the root's key lives in the game's header
 * line and is updated by cz_engine_play) in a device array indexed like the network batch rows.  The reference has no position
 * hashing (nodes are keyed by object identity, main.py:246-247); the keys exist for evaluation de-duplication studies and
 * transposition statistics, they never influence the search.  Capturable; read by waves launched / captured afterwards. */
int cz_engine_enable_hashing(cz_engine *e, int on);
int cz_engine_leaf_hashes(cz_engine *e, uint64_t **dev_keys /* out: device pointer, [n_games*leaves] */);
int cz_engine_root_keys(cz_engine *e, void *stream, uint64_t *keys /* host [B] */);

/* Number of games that still have playouts to run or a leaf pending (device->host, synchronises stream). */
int cz_engine_unfinished(cz_engine *e, void *stream, int32_t *out_count);
/* Asynchronous form: writes the count to *dev_count (device int32) without synchronising. */
int cz_engine_unfinished_async(cz_engine *e, void *stream, int32_t *dev_count);

/* Root statistics in child (= move generation) order: what get_action reads from root.child
 * (main.py:1339) and MCTS_tree.Q (261-270).  HOST buffers; synchronises stream.
 * q = f32(W/N) (0 when N == 0).  Any pointer may be NULL. */
int cz_engine_root_children(cz_engine *e, void *stream, int32_t *n_children /* [B] (-1: root not expanded) */,
                            uint16_t *moves /* [B][128] */, int32_t *visits /* [B][128] */,
                            float *w /* [B][128] */, float *p /* [B][128] */, float *q /* [B][128] */);
/* The root's child count of every game (-1: root not expanded, 0: expanded without children) into HOST counts [B]: one copy of
 * the header lines, synchronises stream. */
int cz_engine_root_counts(cz_engine *e, void *stream, int32_t *counts /* [B] */);
/* Root exploration noise (AlphaZero: P' = (1 - eps) P + eps eta, once per move search; the reference's root Dirichlet is a no-op):
 * for every game with mask[g] != 0 (HOST mask, NULL = all), active (cz_engine_begin_search) and with an expanded root of n > 0
 * children, root prior i becomes f32(keep * f64(P_i) + eps * eta[g][i]) (separately rounded f64 products and sum, no FMA; no
 * renormalisation).  eta: DEVICE f64 [B][128]; *keep is 1 - *eps as the caller computed it, both in [0, 1] (else CZ_EINVAL).  Expand
 * the roots first: cz_engine_begin_search(playouts = 0) and waves until cz_engine_unfinished is 0 expand every pending root and run
 * no playout.  Nothing else in the tree changes; cz_engine_play drops the noised block with the rest of the old root. */
int cz_engine_root_noise(cz_engine *e, void *stream, const uint8_t *mask, const double *eta, const double *keep /* host [1] */,
                         const double *eps /* host [1] */);

/* Play child_index[g] (index into the root's children; < 0 = leave game g alone):
 * GameBoard state update (main.py:1522-1528) + MCTS_tree.update_tree (272-276): the chosen child's
 * subtree is compacted into the other arena half and becomes the root; terminal flags are updated
 * (main.py:1532-1545).  child_index is a HOST buffer. */
int cz_engine_play(cz_engine *e, void *stream, const int32_t *child_index /* [B] */);
/* Same, and returns every game's packed status record (one kernel, one device->host copy, one synchronisation):
 * CZ_STATUS_BYTES per game: [0,90) board | 90 side | 91 terminal (codes of cz_engine_status) | 92 winner (int8) | 96 ply i32 |
 * 100 restrict_round i32 |
 * 104 Q (f32) of the move just played = MCTS_tree.Q(act), main.py:1350 | 108 N of the new root i32. */
#define CZ_STATUS_BYTES 112
int cz_engine_play_status(cz_engine *e, void *stream, const int32_t *child_index /* [B] */, uint8_t *status /* host [B][112] or NULL */);
/* Play a given MOVE in every game (MCTS_tree.update_tree(act) for a move the tree did not choose, human_move main.py:1412-1418 --
 * e.g. the opponent's move in a match where each player keeps its own tree).  moves[g] = src | dst << 7 as cz_engine_root_children
 * returns it, 0xFFFF = leave game g alone.  Expanded root: exactly cz_engine_play of the child that carries the move.  Unexpanded
 * root (fresh reset, or re-rooted onto an unvisited child): the move is checked against the legal moves of the side to move and
 * the game advances to an empty tree at the new position (q = 0; unlike human_move, no search is run first).  A move that is not
 * legal at the root, or any move in a finished game, sets CZ_ERR_ILLEGAL in that game's error word and leaves the game unchanged;
 * the other games are played.  Status records as cz_engine_play_status (q = MCTS_tree.Q(act) of the child played). */
int cz_engine_play_moves(cz_engine *e, void *stream, const uint16_t *moves /* [B] host, 0xFFFF = no move */,
                         uint8_t *status /* host [B][CZ_STATUS_BYTES] or NULL */);
int cz_engine_status_packed(cz_engine *e, void *stream, uint8_t *status /* host [B][112] */);

/* Game status (cchess_main.check_end main.py:1380-1392): HOST buffers, any may be NULL; synchronises.
 * terminal: 0 running, 1 king captured, 2 draw (restrict_round >= 60), 3 mated (strict engines: the side to move has no strictly
 * legal move; the winner is the side that just moved); winner: 0 'w', 1 'b', -1 none. */
int cz_engine_status(cz_engine *e, void *stream, uint8_t *terminal, int8_t *winner, int32_t *ply, int32_t *rr,
                     uint8_t *side, uint8_t *boards /* [B][90] */);

/* Counters since creation, summed over games: out[0] expansions (calls of expand), out[1] playouts,
 * out[2] sum of path lengths L, out[3] sum of scanned children c_l, out[4] OR of per-game error flags,
 * out[5] max arena words in use, out[6] index of first game with an error (or -1), out[7] max path length,
 * out[8] sum over expansions of the number of children C. */
int cz_engine_counters(cz_engine *e, void *stream, int64_t *out /* [9] */);

/* Test hook: flat DFS signature of game g's tree, records of 6 int64
 * (label index, N, W bits, P bits, Q bits, n_children), children in order. Returns record count via *n. */
int cz_engine_tree_signature(cz_engine *e, void *stream, int game, int64_t *out, int64_t cap, int64_t *n);

/* ---- snapshots of games at rest (save / restore a self-play run between plies) ----
 * A game is AT REST when no leaf or root expansion is pending and no playouts are owed (every game after cz_engine_unfinished
 * returned 0, after cz_engine_play, after a reset).  Its whole state is then its 16-word header line, its root board, its five
 * counters, its FIFO event-loop words (cz_engine_create_fifo engines) and words [0, alloc) of its current arena half (the live tree:
 * cz_engine_play compacts it to offset 0).  Blob layout (little-endian, 4-byte words):
 *   head  u64 [6]: magic 0x485350414E535A43 ("CZSNAPSH") | format (low 32 bits: 1 = reference rules, 2 = strict rules, same layout),
 *                  cz_version() (high) | FNV-1a 64 checksum of the
 *                  Zobrist key table | n_games (low), leaves K (high) | narr = arrays per node block, 5 or 6 (low), F (high)
 *   off   i64 [n_games + 1]: word offset of every game's section and of the end; head + off padded to a multiple of 16 bytes
 *   per game: hdr [16] | root board [24] (96 bytes) | counters u64 [5] (expand, playout, L, c, C) | pad [2] | fifo [28] (narr 6
 *             only) | arena [alloc]  -- F = 52 (narr 5) or 80 (narr 6) words precede the arena, alloc = hdr[7]
 * cz_engine_snapshot_size: the blob's size in bytes (synchronises stream).  cz_engine_snapshot: writes it to out (host, cap bytes;
 * *bytes = its size), one pack kernel and one device->host copy.  Both return CZ_EINVAL when a game is not at rest, snapshot also
 * when cap is too small.  cz_engine_restore: validates the whole blob first (cz_snapshot_check_rules against this engine) and returns
 * CZ_EINVAL naming the game and the failed check with the engine untouched; otherwise one host->device copy and one unpack
 * kernel write it IN PLACE into the engine's buffers (captured CUDA graphs stay valid) and every game is at rest.  The arena size
 * may differ from the saving engine's as long as every alloc fits.  Board hashing on / off is not part of a snapshot. */
int cz_engine_snapshot_size(cz_engine *e, void *stream, int64_t *bytes);
int cz_engine_snapshot(cz_engine *e, void *stream, void *out, int64_t cap, int64_t *bytes);
int cz_engine_restore(cz_engine *e, void *stream, const void *in /* host */, int64_t bytes);
/* Host only: the validator restore runs, for an engine of n_games x leaves with narr arrays per block and arena_words per half.
 * Checks magic, format, Zobrist checksum, n_games / leaves / narr; offsets monotone and summing to the blob size; per game: alloc
 * <= arena_words and a multiple of 8, header at rest with valid flag / terminal / winner codes, root child count in {-1, 0..128},
 * root board piece codes 0..14, FIFO loop at rest; every block reachable from the root lies in [0, alloc), 8-word aligned, with a
 * header count equal to its parent's META n_grandchildren and <= 128, blocks disjoint, child pointers above their parent's base,
 * move squares < 90, META bits 24-31 clear.  CZ_OK or CZ_EINVAL (cz_last_error names the game and the check).  This is the check for
 * a reference-rules engine: format 1 only. */
int cz_snapshot_check(const void *in, int64_t bytes, int n_games, int leaves, int narr, int64_t arena_words);
/* The same checks for an engine of the given rules: CZ_RULES_REFERENCE is cz_snapshot_check; CZ_RULES_STRICT accepts format 2 only,
 * where terminal code 3 and mated nodes (an expanded child with n_grandchildren 0, or a root with count 0) may occur, each as a bare
 * 8-word block (the words after it end the tree or start another reachable block).  A blob of the other rules' format is refused
 * ("rules differ").  cz_engine_restore runs this with the engine's rules. */
int cz_snapshot_check_rules(const void *in, int64_t bytes, int n_games, int leaves, int narr, int64_t arena_words, int rules);

/* ---- network ends (policy_value_network.py:45-48 and 55-74), hand-written; the residual tower is library code ----
 * cz_net_first_conv: canonical boards (dev u8 [B][96], from cz_engine_wave with CZ_BOARD) ->
 *     ReLU(conv3x3(14->128) + bias) as fp16 NHWC [B][90][128].  w1: dev fp16 [9 taps][14 pieces][128], b1: dev f32 [128]
 *     (batch norm already folded in).  The one-hot [9][10][14] tensor of main.py:547-557 is never materialised.
 * cz_net_heads: x fp16 [B][90][128] -> logits f32 [B][2086] (raw, no softmax) and value f32 [B] (tanh).
 *     wh f32 [3][128] / bh [3]: 1x1 convs of the policy (2) and value (1) heads with BN folded; w1t f32 [90][256], b1 [256],
 *     w2 [256], b2 [1] (device pointers, so that weights can be refreshed under a captured CUDA graph): value MLP; wp fp16 [2112][192] / bp f32 [2112]: policy FC zero-padded; hp_scratch fp16 [B][192],
 *     hv_scratch f32 [B][96]. */
int cz_net_first_conv(const uint8_t *canon_boards, int B, const void *w1, const float *b1, void *out, void *stream);
int cz_net_heads(const void *x, int B, const float *wh, const float *bh, const float *w1t, const float *b1, const float *w2, const float *b2,
                 const void *wp, const float *bp, void *hp_scratch, float *hv_scratch, float *logits, float *value, void *stream);

/* ---- host side: get_action's sampling for a whole batch of games (main.py:1339-1348), bit-identical to the numpy calls ----
 * For every game g with live[g] != 0 (live NULL = all):  probs = ex[g][:n] / np.sum(ex[g][:n])  (ex = exp(log(visits)/T - max), computed
 * by the caller with numpy);  exploration: p = 0.75 * probs + 0.25 * RandomState.dirichlet(0.3 * ones(n));  choice[g] =
 * RandomState.choice(n, p = p).  mt_states: one legacy MT19937 state per game, CZ_MT_WORDS uint32 each = key[624], pos, 0 --
 * exactly numpy.random.RandomState.get_state()[1:3] -- advanced in place by the same number of draws numpy would make.
 * probs [B][128] receives the normalised (un-noised) probabilities, i.e. the recorded pi.  fallback[g] = 1 when the vector would
 * make numpy raise (NaN / negative / not summing to 1): the caller lets numpy itself handle that game (after the Dirichlet draws,
 * which have been consumed as in the reference).  All pointers are HOST memory; no GPU involved. */
#define CZ_MT_WORDS 626
int cz_host_choose_moves(int n_games, const uint8_t *live, const int32_t *n_children, const double *ex /* [B][128] */, int exploration,
                         uint32_t *mt_states /* [B][626] */, int32_t *choice /* [B] */, double *probs /* [B][128] */, uint8_t *fallback /* [B] */,
                         int n_threads);
/* Root exploration noise, host side: for every game g with mask[g] != 0 (mask NULL = all) and n[g] > 0, eta[g][:n[g]] =
 * RandomState.dirichlet(alpha * ones(n[g])) drawn from mt_states[g] (layout as above), bit-identical to numpy, the state advanced
 * exactly as numpy advances it.  Other games: neither their state nor their eta row is touched.  0 < *alpha < 1 (the shape-below-1
 * branch of numpy's legacy gamma) and n[g] <= 128 for every selected game, else CZ_EINVAL before any draw.  HOST memory only. */
int cz_host_dirichlet(int n_games, const uint8_t *mask, const int32_t *n /* [B] */, const double *alpha /* host [1] */, uint32_t *mt_states /* [B][626] */,
                      double *eta /* [B][128] */, int n_threads);

/* cz_net_heads for large batches: policy FC on wgmma (operands bulk-copied in the K-major no-swizzle layout), 1x1 head convolution on
 * mma.sync, value MLP concurrently.  wp_tiled: dev fp16 [17 label tiles][24 k-chunks][128 labels][8 features] (labels >= 2086 zero),
 * bp f32 [2176]; hp_tiled_scratch: fp16, ceil(B/128) * 49152 bytes, zero-initialised once by the caller. */
int cz_net_heads_tc(const void *x, int B, const float *wh, const float *bh, const float *w1t, const float *b1, const float *w2, const float *b2,
                    const void *wp_tiled, const float *bp, void *hp_tiled_scratch, float *hv_scratch, float *logits, float *value, void *stream);

/* The second half of cz_net_heads alone: value MLP and policy FC on head features that are already computed
 * (hp fp16 [B][192], hv f32 [B][96]) -- what follows cz_net_tower_small. */
int cz_net_heads_fc(const void *hp, const float *hv, int B, const float *w1t, const float *b1, const float *w2, const float *b2,
                    const void *wp, const float *bp, float *logits, float *value, void *stream);

/* ---- the whole convolutional trunk for a FEW positions in one launch (play mode / single-tree search, BASELINE config 5) ----
 * policy_value_network.py:45-74, 151-162 with batch norm folded: first conv3x3(14->128) from the canonical board bytes,
 * n_conv = 2*res_block_nums 3x3 convolutions (residual blocks), the two 1x1 head convolutions; output = the head features
 * hp fp16 [n_pos][192] / hv f32 [n_pos][96] that cz_net_heads_fc turns into logits and value.
 * One thread-block cluster of 4 CTAs per position: activations stay in shared memory (K-major no-swizzle layout,
 * 3x3 taps = descriptor start offsets), weights stream from L2 by TMA, wgmma accumulates in registers, epilogues exchange
 * channel slices through distributed shared memory.  See csrc/cz_tower.cu.
 *   w1     dev fp16 [9][14][128]   (as cz_net_first_conv);  bias dev f32 [1 + n_conv][128];  wh f32 [3][128], bh f32 [3]
 *   wblob  dev fp16, cz_net_tower_blob_bytes(n_conv) bytes, arranged by the CTA that reads each slice:
 *          [conv][tap 9][rank 4][k-chunk 16][out channel 32][8 in channels]   (out channel = 32*rank + row, in channel = 8*chunk + i) */
int64_t cz_net_tower_blob_bytes(int n_conv);
int cz_net_tower_small(const uint8_t *canon_boards, int n_pos, int n_conv, const void *w1, const void *wblob, const float *bias,
                       const float *wh, const float *bh, void *hp, float *hv, void *stream);

/* ---- fp32-accurate inference on the tensor cores (net.py: SplitTf32Plan; policy_value_network.py:202-214 is fp32) ----
 * The split of activations v dev f32 [n_pix][128] (NHWC): hi dev f32 [n_pix][128] = tf32(v) (round to the 10-bit mantissa) and
 * x2 dev fp16 [n_pix][256] = { (v - hi) * 2^11 | hi } (both exact in fp16).  A TF32 convolution of hi with hi(w) and an fp16
 * convolution of x2 with { hi(w) | lo(w) * 2^11 } accumulate hi*hi and (lo*hi + hi*lo) * 2^11 in two separate f32 chains (the
 * tensor cores' accumulator truncates, measured -6.6e-9 relative per accumulated term: the full-size terms get the short chain).
 * cz_net_epilogue_split is the f32 epilogue of such a convolution fused with the split for the next one, one streaming pass:
 *   v = ReLU(t + 2^-11 s + bias [+ skip]);   x = v (optional);   hi, x2 = split of v (optional, both or neither)
 * t dev f32 [n_pix][128] (hi*hi, raw); s dev fp16 [n_pix][128] or NULL (cross terms, raw, scaled by 2^11); bias dev f32 [128];
 * skip dev f32 [n_pix][128] or NULL (x may alias skip). */
int cz_net_epilogue_split(const float *t, const void *s, const float *bias, const float *skip, float *x, float *hi, void *x2, long long n_pix, void *stream);

#ifdef __cplusplus
}
#endif
#endif
