"""Tiny end-to-end run for compute-sanitizer (memcheck / racecheck / initcheck): rules, waves in every dtype, re-root."""
import sys
sys.path.insert(0, '.')
import numpy as np, torch
from cchess_zero_b200 import rules
from cchess_zero_b200.fakenet import FakeNet
from cchess_zero_b200.selfplay import SelfPlay
from cchess_zero_b200.net import policy_value_network

rules._init_tables()
b = rules.state_to_board(rules.START_STATE)
mv, cnt = rules.legal_moves_batch(np.stack([b] * 5), [0, 1, 0, 1, 0])
enc = rules.encode_batch(np.stack([b] * 5), [0, 1, 0, 1, 0])
nb, cap = rules.apply_moves_batch(np.stack([b] * 2), mv[0, :2])
sp = SelfPlay(8, FakeNet("hash_pos"), 24, seeds=range(8), arena_words=1 << 16, auto_reset=True)
for _ in range(4):
    sp.step()
sp.engine.raise_on_error()
pv = policy_value_network(res_block_nums=1)
sp2 = SelfPlay(8, None, 16, seeds=range(8), arena_words=1 << 16, plan=pv.native_plan(8))
for _ in range(3):
    sp2.step()
sp2.engine.raise_on_error()
print("sanitize run ok", cnt[:2], enc.sum(), sp.plies, sp2.plies)
# round 2: the search_threads = K event-loop kernel, the leaf-parallel kernel, hashing, and the cluster trunk
sp3 = SelfPlay(4, FakeNet("hash_pos"), 48, seeds=range(4), arena_words=1 << 16, auto_reset=True, search_threads=16)
for _ in range(3):
    sp3.step()
sp3.engine.raise_on_error()
sp4 = SelfPlay(8, FakeNet("hash_signed"), 24, seeds=range(8), arena_words=1 << 16, auto_reset=True, hashing=True)
for _ in range(3):
    sp4.step()
sp4.engine.raise_on_error()
from cchess_zero_b200.mcts import MCTS_tree
t = MCTS_tree(rules.START_STATE, pv.forward, 1, leaf_parallel=4)
t.main(rules.START_STATE, "w", 0, 32)
boards = torch.zeros((3, 96), dtype=torch.uint8, device="cuda"); boards[:, :90] = torch.from_numpy(np.stack([b] * 3)).cuda()
lo = torch.zeros((3, 2086), device="cuda"); vo = torch.zeros((3,), device="cuda")
pv.small_plan(4)(boards, lo, vo)
torch.cuda.synchronize()
print("round-2 kernels ok", sp3.plies, sp4.plies, float(lo.abs().max()))
# later in round 2: row compaction of the K-thread batch (sp3 above runs through cz_engine_wave_compact by default), the tf32x3 plan
# (k_epilogue_split + library convolutions), the single-tree graph with several waves per replay
assert sp3.compact and sp3.rows_evaluated > 0
pv3 = policy_value_network(res_block_nums=1, precision="tf32x3")
x = torch.zeros((3, 9, 10, 14), device="cuda"); x[:, :, :, 2] = 1.0
l3, v3 = pv3.plan()(x)
t2 = MCTS_tree(rules.START_STATE, pv.forward, 1)
t2.main(rules.START_STATE, "w", 0, 20)
torch.cuda.synchronize()
print("later round-2 kernels ok", sp3.rows_evaluated, float(l3.abs().max()), t2._reps)
