"""Device time of the hand-written network-end kernels at the bench batch (CUDA events, 300 back-to-back launches each, warm)."""
import contextlib, io, json, sys
sys.path.insert(0, '.')
import ctypes as C
import torch
from cchess_zero_b200.net import policy_value_network

B = int(sys.argv[1]) if len(sys.argv) > 1 else 1024
with contextlib.redirect_stdout(io.StringIO()):
    pv = policy_value_network(7, precision="fp16")
plan = pv.native_plan(B)
lib = plan._lib
boards = torch.zeros((B, 96), dtype=torch.uint8, device="cuda")
boards[:, :90] = (torch.randint(1, 15, (B, 90), device="cuda") * (torch.rand((B, 90), device="cuda") < 0.3)).to(torch.uint8)
x = torch.randn((B, 9, 10, 128), device="cuda").clamp_(min=0).half()
lo = torch.zeros((B, 2086), device="cuda"); vo = torch.zeros((B,), device="cuda")
st = C.c_void_p(torch.cuda.current_stream().cuda_stream)


def timed(fn, n=300):
    """fn captured into a CUDA graph and replayed: device time without the host's launch cost."""
    for _ in range(5):
        fn()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        global st
        st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
        fn()
        torch.cuda.synchronize()
        with torch.cuda.graph(g, stream=s):
            st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
            for _ in range(10):
                fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    g.replay()
    e0.record()
    for _ in range(n // 10):
        g.replay()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e3 / (n // 10 * 10)


out = {}
out["first_conv_gather_us"] = timed(lambda: lib.cz_net_first_conv(boards.data_ptr(), B, plan.w1.data_ptr(), plan.b1.data_ptr(), plan.x1.data_ptr(), st))
heads = lambda: lib.cz_net_heads(x.data_ptr(), B, plan.wh.data_ptr(), plan.bh.data_ptr(), plan.w1t.data_ptr(), plan.bv1.data_ptr(), plan.w2.data_ptr(),
                                 plan.b2t.data_ptr(), plan.wp.data_ptr(), plan.bp.data_ptr(), plan.hp.data_ptr(), plan.hv.data_ptr(), lo.data_ptr(), vo.data_ptr(), st)
out["heads_all_us"] = timed(heads)
out["heads_fc_only_us"] = timed(lambda: lib.cz_net_heads_fc(plan.hp.data_ptr(), plan.hv.data_ptr(), B, plan.w1t.data_ptr(), plan.bv1.data_ptr(), plan.w2.data_ptr(),
                                                             plan.b2t.data_ptr(), plan.wp.data_ptr(), plan.bp.data_ptr(), lo.data_ptr(), vo.data_ptr(), st))
out["heads_tc_all_us"] = timed(lambda: lib.cz_net_heads_tc(x.data_ptr(), B, plan.wh.data_ptr(), plan.bh.data_ptr(), plan.w1t.data_ptr(), plan.bv1.data_ptr(), plan.w2.data_ptr(),
                                                           plan.b2t.data_ptr(), plan.wp_tiled.data_ptr(), plan.bp_pad.data_ptr(), plan.hp_tiled.data_ptr(), plan.hv.data_ptr(),
                                                           lo.data_ptr(), vo.data_ptr(), st))
out["head_conv_us"] = out["heads_all_us"] - out["heads_fc_only_us"]
print(json.dumps(dict(batch=B, **out)))
