"""Per-section device time of one wave (CUDA events, eager launches, warm state): k_wave / first conv / tower / heads."""
import sys, json
sys.path.insert(0, '.')
import numpy as np, torch, ctypes as C
from cchess_zero_b200.net import policy_value_network
from cchess_zero_b200.selfplay import SelfPlay

B = int(sys.argv[1]) if len(sys.argv) > 1 else 1024
plies = int(sys.argv[2]) if len(sys.argv) > 2 else 6
pv = policy_value_network(7, precision="fp16")
plan = pv.native_plan(B)
sp = SelfPlay(B, None, 1200, seeds=range(B), plan=plan)
sp.capture_graph()
for _ in range(plies):
    sp.step()
e = sp.engine
e.begin_search(1200)
lib = plan._lib
def ev(): return torch.cuda.Event(enable_timing=True)
sections = {k: [] for k in ("k_wave", "first_conv", "tower", "heads")}
st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
for it in range(300):
    t = [ev() for _ in range(5)]
    t[0].record()
    e.wave(sp.nn_in, sp.logits, sp.value)
    t[1].record()
    lib.cz_net_first_conv(sp.nn_in.data_ptr(), B, plan.w1.data_ptr(), plan.b1.data_ptr(), plan.x1.data_ptr(), st)
    t[2].record()
    x = plan.x1[:B].permute(0, 3, 1, 2)
    for c1, c2 in plan.blocks:
        y = plan._base._conv_relu(x, c1, 1)
        x = plan._base._conv_add_relu(y, c2, x)
    t[3].record()
    lib.cz_net_heads(x.data_ptr(), B, plan.wh.data_ptr(), plan.bh.data_ptr(), plan.w1t.data_ptr(), plan.bv1.data_ptr(), plan.w2.data_ptr(), plan.b2t.data_ptr(),
                     plan.wp.data_ptr(), plan.bp.data_ptr(), plan.hp.data_ptr(), plan.hv.data_ptr(), sp.logits.data_ptr(), sp.value.data_ptr(), st)
    t[4].record()
    if it >= 50:
        sections["_ev"] = sections.get("_ev", []) + [t]
torch.cuda.synchronize()
for t in sections.pop("_ev"):
    for i, k in enumerate(("k_wave", "first_conv", "tower", "heads")):
        sections[k].append(t[i].elapsed_time(t[i + 1]) * 1e3)
out = {k: dict(mean_us=float(np.mean(v)), p50=float(np.median(v)), p90=float(np.percentile(v, 90)), max=float(np.max(v))) for k, v in sections.items()}
out["sum_mean_us"] = sum(v["mean_us"] for v in out.values())
# graph replay of the whole wave for comparison
g0, g1 = ev(), ev()
g0.record()
for _ in range(200): sp.graph.replay()
g1.record(); torch.cuda.synchronize()
out["graph_wave_us"] = g0.elapsed_time(g1) / 200 * 1e3
# tower alone in a graph
xb = plan.x1[:B].permute(0, 3, 1, 2)
def tower():
    x = xb
    for c1, c2 in plan.blocks:
        y = plan._base._conv_relu(x, c1, 1)
        x = plan._base._conv_add_relu(y, c2, x)
    return x
s = torch.cuda.Stream(); s.wait_stream(torch.cuda.current_stream())
with torch.cuda.stream(s):
    tower()
torch.cuda.current_stream().wait_stream(s)
g = torch.cuda.CUDAGraph()
with torch.cuda.graph(g):
    tower()
g0.record()
for _ in range(200): g.replay()
g1.record(); torch.cuda.synchronize()
out["graph_tower_us"] = g0.elapsed_time(g1) / 200 * 1e3
print(json.dumps(out))
