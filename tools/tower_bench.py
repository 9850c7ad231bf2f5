"""Per-call device time (CUDA events, warm L2, 200 calls) of the network evaluation at small batch: the one-launch cluster trunk
(csrc/cz_tower.cu) vs the library trunk (cuDNN convs + csrc/cz_net.cu ends), eager and inside a CUDA graph."""
import contextlib, io, json, sys
sys.path.insert(0, '.')
import torch
from cchess_zero_b200.net import policy_value_network

blocks = int(sys.argv[1]) if len(sys.argv) > 1 else 7
with contextlib.redirect_stdout(io.StringIO()):
    pv = policy_value_network(res_block_nums=blocks)
out = {}
for B in (1, 8, 16):
    boards = torch.zeros((B, 96), dtype=torch.uint8, device="cuda")
    boards[:, :90] = torch.randint(0, 15, (B, 90), dtype=torch.uint8, device="cuda") * (torch.rand((B, 90), device="cuda") < 0.3)
    lo = torch.zeros((B, 2086), device="cuda"); vo = torch.zeros((B,), device="cuda")
    plans = {"library_trunk": pv.native_plan(B), "cluster_trunk": pv.small_plan(B)}
    for name, plan in plans.items():
        for _ in range(5):
            plan(boards, lo, vo)
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        s = torch.cuda.Stream()
        with torch.cuda.stream(s):
            plan(boards, lo, vo)
            torch.cuda.synchronize()
            with torch.cuda.graph(g, stream=s):
                plan(boards, lo, vo)
        res = {}
        for mode in ("eager", "graph"):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            e0.record()
            for _ in range(200):
                g.replay() if mode == "graph" else plan(boards, lo, vo)
            e1.record()
            torch.cuda.synchronize()
            res[mode + "_us"] = e0.elapsed_time(e1) * 1e3 / 200
        out["B%d_%s" % (B, name)] = res
print(json.dumps(dict(res_block_nums=blocks, per_call_us=out), indent=1))
