"""wgmma flash-attention forward vs the library SDPA (cuDNN / flash) on the Llama-3-8B attention shape."""
import json

import torch
import torch.nn.functional as F

from colossalai_b200.ops import flash_attn_native as fa


def timeit(fn, iters=20):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(iters):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / iters


for (B, S, Hq, Hkv, D) in [(1, 4096, 32, 8, 128), (4, 4096, 32, 8, 128), (1, 16384, 32, 8, 128)]:
    q = torch.randn(B * S, Hq, D, device="cuda", dtype=torch.bfloat16)
    k = torch.randn(B * S, Hkv, D, device="cuda", dtype=torch.bfloat16)
    v = torch.randn(B * S, Hkv, D, device="cuda", dtype=torch.bfloat16)
    qb, kb, vb = (t.view(B, S, -1, D).transpose(1, 2) for t in (q, k, v))
    t_nat = timeit(lambda: fa.flash_fwd(q, k, v, B, True, None))
    t_lib = timeit(lambda: F.scaled_dot_product_attention(qb, kb, vb, is_causal=True, enable_gqa=True))
    fl = 4.0 * B * Hq * S * S * D / 2
    print("FLASH_FWD " + json.dumps({"B": B, "S": S, "Hq": Hq, "Hkv": Hkv, "D": D, "native_ms": t_nat, "sdpa_ms": t_lib,
                                     "native_tflops": fl / t_nat / 1e9, "sdpa_tflops": fl / t_lib / 1e9}), flush=True)
    # backward: ours = one launch chain (delta, wgmma bwd, dq cast); library = autograd through SDPA (cuDNN bprop)
    out, lse = fa.flash_fwd(q, k, v, B, True, None)
    dout = torch.randn_like(out)
    t_nat_b = timeit(lambda: fa.flash_bwd(q, k, v, out, dout, lse, B, True, None))
    ql, kl, vl = (t.detach().clone().requires_grad_(True) for t in (qb, kb, vb))
    ol = F.scaled_dot_product_attention(ql, kl, vl, is_causal=True, enable_gqa=True)
    gl = torch.randn_like(ol)
    t_lib_b = timeit(lambda: torch.autograd.grad(ol, (ql, kl, vl), gl, retain_graph=True))
    print("FLASH_BWD " + json.dumps({"B": B, "S": S, "Hq": Hq, "Hkv": Hkv, "D": D, "native_ms": t_nat_b,
                                     "sdpa_ms": t_lib_b, "native_tflops": 2.5 * fl / t_nat_b / 1e9,
                                     "sdpa_tflops": 2.5 * fl / t_lib_b / 1e9}), flush=True)
