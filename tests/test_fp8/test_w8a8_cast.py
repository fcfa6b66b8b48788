"""A floating-point cast of a SmoothQuant `W8A8Linear` (as the inference engine does with `model.to(dtype)`) keeps its
per-channel weight scales and static activation scale in fp32 and its weight in int8, so the layer computes the same
function before and after the cast."""
import torch
import torch.nn as nn

from colossalai_b200.quantization.smoothquant import W8A8Linear


def test_cast_keeps_w8a8_scales_fp32():
    torch.manual_seed(0)
    lin = nn.Linear(64, 32, bias=False)           # a bias is a parameter: a cast rounds it like any other
    lin.weight.data[:, 0] *= 3.3                # scales that bf16 would round
    q = W8A8Linear.from_float(lin, "static", act_absmax=7.7)
    ws, act = q.weight_scale.clone(), q.act_scale.clone()
    x = torch.randn(5, 64)
    before = q(x)
    for dtype in (torch.bfloat16, torch.float16, torch.float64):
        q.to(dtype)
        assert q.weight_scale.dtype == torch.float32 and q.act_scale.dtype == torch.float32
        assert torch.equal(q.weight_scale, ws) and torch.equal(q.act_scale, act)
        assert q.weight.dtype == torch.int8
        q.float()
    assert torch.equal(q(x), before)
    assert not torch.equal(ws.bfloat16().float(), ws)   # the cast would have changed the scales
