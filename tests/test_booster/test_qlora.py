"""QLoRA through the Booster: `enable_lora(..., bnb_quantization_config=...)` quantises the targeted linears into packed
nf4 / fp4 / int8 layers, wraps them with LoRA adapters, and only the adapters train (DDP and ZeRO-2 bf16, two gloo
ranks).  The packed base stays bitwise frozen, its quantisation state stays fp32 through the plugin's precision cast,
the adapter gradients match a float64 model on the dequantised weights, and saved adapters reload into a freshly
quantised model."""
import copy
import os

import pytest
import torch
import torch.distributed as dist
import torch.nn as nn

import colossalai_b200
from colossalai_b200.booster import Booster
from colossalai_b200.booster.lora import LoraConfig, LoraLinear
from colossalai_b200.booster.plugin import LowLevelZeroPlugin, TorchDDPPlugin
from colossalai_b200.models import build_model
from colossalai_b200.quantization import BnbQuantizationConfig
from colossalai_b200.quantization.bnb import Linear4bit, Linear8bit
from colossalai_b200.testing import rerun_if_address_is_in_use, spawn

TARGETS = ["qkv_proj", "o_proj", "gate_up_proj", "down_proj"]
FORMATS = {
    "nf4": dict(load_in_4bit=True, bnb_4bit_quant_type="nf4"),
    "fp4": dict(load_in_4bit=True, bnb_4bit_quant_type="fp4"),
    "nf4_dq": dict(load_in_4bit=True, bnb_4bit_quant_type="nf4", bnb_4bit_use_double_quant=True),
    "int8": dict(load_in_8bit=True),
}


def _cfg(fmt, compute):
    kw = dict(FORMATS[fmt])
    if fmt == "int8":
        kw["torch_dtype"] = {"fp32": torch.float32, "bf16": torch.bfloat16}[compute]
    else:
        kw["bnb_4bit_compute_dtype"] = compute
    return BnbQuantizationConfig(**kw)


def _unwrap(model):
    inner = model.unwrap() if hasattr(model, "unwrap") else model
    return inner.module if hasattr(inner, "module") and not hasattr(inner, "cfg") else inner


def _packed(model):
    return {n: b.detach().clone() for n, b in model.named_buffers() if n.endswith(("packed", "weight_q", "absmax_q"))}


def _float64_reference(model):
    """The model in float64 with every quantised base replaced by an nn.Linear holding its dequantised weight."""
    ref = copy.deepcopy(model)
    for m in ref.modules():
        if isinstance(m, LoraLinear) and isinstance(m.base_layer, (Linear4bit, Linear8bit)):
            q = m.base_layer
            lin = nn.Linear(q.in_features, q.out_features, bias=q.bias is not None)
            lin.weight.data = q.dequantize().double()
            if q.bias is not None:
                lin.bias.data = q.bias.detach().double()
            m.base_layer = lin.requires_grad_(False)
    return ref.double()


def _run(plugin, fmt, compute, tmp, tag):
    torch.manual_seed(0)
    model = build_model("llama-tiny")
    booster = Booster(plugin=plugin)
    lcfg = LoraConfig(r=4, lora_alpha=8, target_modules=TARGETS)
    model = booster.enable_lora(model, lora_config=lcfg, bnb_quantization_config=_cfg(fmt, compute))
    qtype = Linear8bit if fmt == "int8" else Linear4bit
    wrapped = [m for m in model.modules() if isinstance(m, LoraLinear)]
    assert len(wrapped) == len(TARGETS) * model.cfg.num_hidden_layers, tag
    assert all(isinstance(m.base_layer, qtype) for m in wrapped), tag
    trainable = {n for n, p in model.named_parameters() if p.requires_grad}
    assert trainable and all(".lora_A." in n or ".lora_B." in n for n in trainable), (tag, trainable)
    assert len(trainable) == 2 * len(wrapped)

    opt = torch.optim.AdamW([p for p in model.parameters() if p.requires_grad], lr=2e-2)
    model, opt, *_ = booster.boost(model, opt)
    inner = _unwrap(model)
    before = _packed(inner)
    for name, buf in inner.named_buffers():
        if name.endswith(("absmax", "scale", "code", "absmax_meta")):
            assert buf.dtype == torch.float32, (tag, name, buf.dtype)

    ids = (torch.arange(32)[None] * 3 + torch.tensor([[1], [5]])) % 512     # the same batch on both ranks
    if isinstance(plugin, TorchDDPPlugin):
        # one step's adapter gradients against float64 on the dequantised weights
        ref = _float64_reference(inner)
        ref(input_ids=ids, labels=ids)["loss"].backward()
        loss = model(input_ids=ids, labels=ids)["loss"]
        booster.backward(loss, opt)
        got = {n: p.grad for n, p in inner.named_parameters() if p.requires_grad}
        want = {n: p.grad for n, p in ref.named_parameters() if p.requires_grad}
        assert got.keys() == want.keys()
        for n, g in got.items():
            w = want[n]
            tol = 1e-4 if compute == "fp32" else 3e-2
            err = (g.double() - w).abs().max().item()
            assert err <= tol * w.abs().max().item() + 1e-7, (tag, n, err, w.abs().max().item())
        opt.step()
        opt.zero_grad()
    losses = []
    for _ in range(4):
        loss = model(input_ids=ids, labels=ids)["loss"]
        booster.backward(loss, opt)
        opt.step()
        opt.zero_grad()
        losses.append(float(loss))
    assert losses[-1] < losses[0], (tag, losses)
    after = _packed(inner)
    assert before.keys() == after.keys() and before
    for n in before:
        assert torch.equal(before[n], after[n]), (tag, n)

    path = os.path.join(tmp, tag)
    booster.save_lora_as_pretrained(model, path)
    dist.barrier()
    torch.manual_seed(0)
    fresh = booster.enable_lora(build_model("llama-tiny"), pretrained_dir=path,
                                bnb_quantization_config=_cfg(fmt, compute))
    fresh = fresh.to(next(inner.parameters()).dtype)
    probe = torch.randint(0, 512, (1, 16), generator=torch.Generator().manual_seed(9))
    inner.eval()
    with torch.no_grad():
        want = inner(input_ids=probe)["logits"].float()
        got = fresh.eval()(input_ids=probe)["logits"].float()
    torch.testing.assert_close(got, want, atol=1e-5, rtol=1e-5, msg=lambda m: f"{tag}: {m}")
    with pytest.raises(NotImplementedError):
        next(m for m in fresh.modules() if isinstance(m, LoraLinear)).merge()


def _worker(rank, world_size, port, tmp):
    colossalai_b200.launch(rank, world_size, "127.0.0.1", port, backend="gloo", verbose=False)
    for fmt in FORMATS:
        _run(TorchDDPPlugin(), fmt, "fp32", tmp, f"ddp_{fmt}")
        _run(LowLevelZeroPlugin(stage=2, precision="bf16"), fmt, "bf16", tmp, f"zero2_bf16_{fmt}")
    dist.destroy_process_group()


@pytest.mark.dist
@rerun_if_address_is_in_use()
def test_qlora_through_booster_plugins(tmp_path):
    spawn(_worker, 2, tmp=str(tmp_path))
