"""One evaluation by the cluster trunk (for ncu): python tools/tower_probe.py [blocks]"""
import contextlib, io, sys
sys.path.insert(0, '.')
import torch
from cchess_zero_b200.net import policy_value_network
blocks = int(sys.argv[1]) if len(sys.argv) > 1 else 7
with contextlib.redirect_stdout(io.StringIO()):
    pv = policy_value_network(res_block_nums=blocks)
plan = pv.small_plan(1)
boards = torch.zeros((1, 96), dtype=torch.uint8, device="cuda")
lo = torch.zeros((1, 2086), device="cuda"); vo = torch.zeros((1,), device="cuda")
for _ in range(30):
    plan(boards, lo, vo)
torch.cuda.synchronize()
print("ok")
