"""Timing of the wgmma layers against cuBLAS on the same box (not the bench contract): python tools/perf_nn.py [envs]
Every variant is captured into a CUDA graph and replayed (that is how the step uses it); times are CUDA events over 50 replays."""
import os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch
from vid2player3d_b200 import nn

M = int(sys.argv[1]) if len(sys.argv) > 1 else 8192
dev = "cuda:0"


def graph_ms(fn, reps=50):
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(3):
            fn()
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        fn()
    g.replay()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        g.replay()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


net = nn.PolicyMLP.random(M, dev)
obs = torch.randn(M, 734, device=dev)
ms = graph_ms(lambda: net(obs))
print(f"PolicyMLP b200nn (cast + 4 wgmma launches): {ms * 1e3:.1f} us  {net.flops / ms / 1e9:.1f} TFLOP/s")
for i, l in enumerate(net.layers):
    t = graph_ms(l.run)
    print(f"   layer {i}: {t * 1e3:.1f} us  {l.flops / t / 1e9:.1f} TFLOP/s")

dims = [734, 1024, 1024, 512, 75]
for dt, name, tf32 in ((torch.float32, "torch fp32 (no tf32)", False), (torch.float32, "torch fp32 (tf32 allowed)", True), (torch.bfloat16, "torch bf16 (cuBLAS)", False)):
    torch.backends.cuda.matmul.allow_tf32 = tf32
    mods = []
    for i in range(4):
        mods.append(torch.nn.Linear(dims[i], dims[i + 1]))
        if i < 3:
            mods.append(torch.nn.ReLU())
    ref = torch.nn.Sequential(*mods).to(dev, dt)
    x = obs.to(dt)

    def f():
        with torch.no_grad():
            return ref(torch.clamp(obs, -5, 5).to(dt)).float()
    t = graph_ms(f)
    print(f"{name}: {t * 1e3:.1f} us  {net.flops / t / 1e9:.1f} TFLOP/s")
torch.backends.cuda.matmul.allow_tf32 = False

dec = nn.MixedDecoder.random(M, dev)
z, c = torch.randn(M, 32, device=dev), torch.randn(M, 288, device=dev)
t = graph_ms(lambda: dec(z, c))
print(f"MixedDecoder b200nn ({dec.launches_per_forward} launches): {t * 1e3:.1f} us  {dec.flops / t / 1e9:.1f} TFLOP/s")
for name, l in (("gate1", dec.gate1), ("gate2", dec.gate2), ("l1", dec.l1), ("l2", dec.l2), ("l3", dec.l3)):
    tt = graph_ms(l.run)
    print(f"   {name}: {tt * 1e3:.1f} us  {l.flops / tt / 1e9:.1f} TFLOP/s")
# the reference formulation (per-env blended weights + baddbmm), bf16 autocast like motion_vae/base.py:390-406, at a batch that fits
ws = [torch.randn(6, i, o, device=dev) * 0.05 for i, o in ((320, 256), (288, 256), (288, 290))]
bs = [torch.zeros(6, o, device=dev) for o in (256, 256, 290)]
coef = torch.softmax(torch.randn(M, 6, device=dev), 1)


def ref_moe():
    with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
        h = c
        for i, (w, b) in enumerate(zip(ws, bs)):
            mixed_w = torch.matmul(coef, w.flatten(1, 2)).view(M, *w.shape[1:3])
            inp = torch.cat((z, h), 1).unsqueeze(1)
            mixed_b = torch.matmul(coef, b).unsqueeze(1)
            h = torch.baddbmm(mixed_b, inp, mixed_w).squeeze(1)
            if i < 2:
                h = torch.nn.functional.elu(h)
        return h
try:
    t = graph_ms(ref_moe, reps=10)
    print(f"MixedDecoder reference formulation (per-env blended weights + baddbmm, autocast bf16): {t * 1e3:.1f} us")
except Exception as ex:
    print("reference formulation failed:", repr(ex)[:200])
