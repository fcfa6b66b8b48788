"""Policy that shards a user's HuggingFace Mixtral in place: tensor-parallel attention + EXPERT-PARALLEL experts
(reference `policies/mixtral.py:30-250` + `modeling/mixtral.py:50-210` `EPMixtralSparseMoeBlock`).

transformers >= 5 keeps all experts of a layer in one module (`MixtralExperts`: `gate_up_proj [E, 2 I, H]`,
`down_proj [E, H, I]`) with the interface `forward(hidden_states [T, H], top_k_index [T, k], top_k_weights [T, k])`.
That is exactly the contract of this framework's MoE data path, so the policy
  * keeps only the LOCAL experts' slices of the two parameters on every rank of `shard_config.ep_group`
    (parameter replacement; the slices are tagged so that checkpoints gather them), and
  * rebinds `MixtralExperts.forward` to `moe.dispatch_combine.moe_forward`: dropless dispatch to the owners (fused
    NVLink dispatch on sm_90a, uneven all-to-all elsewhere), grouped per-expert GEMMs on the local slices, SwiGLU,
    combine with the routing weights;
the router (`gate`) stays replicated.  Attention is tensor-parallel like the llama-likes when TP is enabled.  Expert
gradients are already sums over every token of the expert-parallel group that chose the expert; the usual 1 / ep scaling
for data-parallel averaging is the plugin's job (`MoeHybridParallelPlugin`).  Pipeline stages work as for the llama-likes
(`HFDecoderPipelineMixin`): the backbone has the same `embed_tokens / layers / norm` layout."""
from __future__ import annotations

from typing import Dict, List

import torch
import torch.nn as nn

from ..layer import Linear1D_Col, Linear1D_Row, VocabParallelEmbedding1D, VocabParallelLMHead1D
from .base_policy import ModulePolicyDescription, Policy, SubModuleReplacementDescription
from .hf_decoder import HFDecoderPipelineMixin, _fused_rmsnorm_forward, mark_head_norms

__all__ = ["HFMoEPolicy", "HFMixtralPolicy", "HFQwen3MoePolicy", "HFQwen2MoePolicy", "HFDeepseekV3Policy",
           "HFDeepseekV2Policy"]


def _ep_experts_forward(self, hidden_states: torch.Tensor, top_k_index: torch.Tensor, top_k_weights: torch.Tensor):
    from ... import ops
    from ...moe.dispatch_combine import moe_forward
    from ...moe.grouped_gemm import grouped_linear

    act = getattr(self, "_cb200_act", "silu")

    def experts(rows: torch.Tensor, counts: torch.Tensor) -> torch.Tensor:
        h = grouped_linear(rows, self.gate_up_proj, counts)
        h = ops.glu(h, act, valid_rows=counts.sum())
        return grouped_linear(h, self.down_proj, counts)

    shape = hidden_states.shape
    x = hidden_states.reshape(-1, shape[-1])
    out = moe_forward(x, top_k_weights.reshape(x.shape[0], -1).float(), top_k_index.reshape(x.shape[0], -1), experts,
                      self._cb200_num_experts, self._cb200_ep_group)
    return out.to(hidden_states.dtype).reshape(shape)


class HFMoEPolicy(HFDecoderPipelineMixin, Policy):
    """Shared implementation: the HF MoE families of transformers >= 5 all use the same experts module contract
    (`gate_up_proj [E, 2 I, H]`, `down_proj [E, H, I]`, `forward(hidden_states, top_k_index, top_k_weights)`); a family
    is described by its class-name prefix, the name of its experts class and whether its attention is the plain
    q / k / v / o layout that the tensor-parallel replacement understands."""

    FAMILY = "Mixtral"
    EXPERTS_CLASS = "MixtralExperts"
    TP_ATTENTION = True
    NUM_EXPERTS_ATTR = "num_local_experts"

    def config_sanity_check(self) -> None:
        cfg, sc = self.model.config, self.shard_config
        if sc.enable_tensor_parallelism:
            assert self.TP_ATTENTION, (f"tensor parallelism of HF {self.FAMILY} attention (multi-head latent attention) is "
                                       "not provided in place: use expert parallelism only, or the native zoo")
            assert cfg.num_attention_heads % sc.tensor_parallel_size == 0 and \
                cfg.num_key_value_heads % sc.tensor_parallel_size == 0, "attention heads must be divisible by the TP size"
        if sc.ep_group is not None:
            assert getattr(cfg, self.NUM_EXPERTS_ATTR) % sc.expert_parallel_size == 0, \
                "experts must be divisible by the EP size"
        assert not sc.enable_sequence_parallelism, \
            "sequence parallelism of HF modules is not supported; build the model from the native zoo (models.hf_io)"

    def preprocess(self) -> nn.Module:
        self.tie_weight = self.tie_weight_check()
        return self.model

    def postprocess(self) -> nn.Module:
        sm = self.pipeline_stage_manager
        single_stage = sm is None or sm.num_stages == 1
        if getattr(self, "tie_weight", False) and self.shard_config.enable_tensor_parallelism and single_stage:
            emb, head = self.model.get_input_embeddings(), self.model.get_output_embeddings()
            if head is not None and emb is not None and head.weight.shape == emb.weight.shape:
                head.weight = emb.weight
        self._install_pipeline_stage()                      # 1F1B stages: same backbone layout as the llama-likes
        return self.model

    def _slice_experts(self, module: nn.Module) -> None:
        from ...parallel import comm
        from ...tensor.d_tensor.api import mark_sharded, sharded_tensor_to_param

        group = self.shard_config.ep_group
        ep, rank = comm.group_size(group), comm.group_rank(group)
        n_local = module.num_experts // ep
        for name in ("gate_up_proj", "down_proj"):
            full = getattr(module, name).data
            local = full[rank * n_local:(rank + 1) * n_local].clone()
            setattr(module, name, sharded_tensor_to_param(mark_sharded(local, 0, group)))
        module._cb200_num_experts = module.num_experts
        module._cb200_ep_group = group
        module._cb200_act = getattr(self.model.config, "hidden_act", "silu")
        module.num_experts_local = n_local

    def module_policy(self) -> Dict[str, ModulePolicyDescription]:
        sc = self.shard_config
        policy: Dict[str, ModulePolicyDescription] = {}
        if sc.enable_tensor_parallelism:
            fp8 = dict(fp8_communication=sc.fp8_communication)
            vocab = dict(make_vocab_size_divisible_by=sc.make_vocab_size_divisible_by, fp8_communication=sc.fp8_communication)
            policy[f"{self.FAMILY}DecoderLayer"] = ModulePolicyDescription(sub_module_replacement=[
                SubModuleReplacementDescription("self_attn.q_proj", Linear1D_Col, kwargs=dict(fp8)),
                SubModuleReplacementDescription("self_attn.k_proj", Linear1D_Col, kwargs=dict(fp8)),
                SubModuleReplacementDescription("self_attn.v_proj", Linear1D_Col, kwargs=dict(fp8)),
                SubModuleReplacementDescription("self_attn.o_proj", Linear1D_Row, kwargs=dict(fp8)),
            ])
            policy[f"{self.FAMILY}Attention"] = ModulePolicyDescription(
                param_replacement=[mark_head_norms(sc.tensor_parallel_process_group)])
            policy[f"{self.FAMILY}Model"] = ModulePolicyDescription(sub_module_replacement=[
                SubModuleReplacementDescription("embed_tokens", VocabParallelEmbedding1D, kwargs=vocab)])
            policy[f"{self.FAMILY}ForCausalLM"] = ModulePolicyDescription(sub_module_replacement=[
                SubModuleReplacementDescription("lm_head", VocabParallelLMHead1D, kwargs=dict(gather_output=True, **vocab))])
        if sc.ep_group is not None and sc.expert_parallel_size > 1:
            policy[self.EXPERTS_CLASS] = ModulePolicyDescription(param_replacement=[self._slice_experts],
                                                               method_replacement={"forward": _ep_experts_forward})
        if sc.enable_fused_normalization:
            policy[f"{self.FAMILY}RMSNorm"] = ModulePolicyDescription(method_replacement={"forward": _fused_rmsnorm_forward})
        return policy


class HFMixtralPolicy(HFMoEPolicy):
    """`MixtralModel`, `MixtralForCausalLM`."""


class HFQwen3MoePolicy(HFMoEPolicy):
    """`Qwen3MoeModel`, `Qwen3MoeForCausalLM` (per-head q / k norms stay replicated: they act on head_dim)."""
    FAMILY, EXPERTS_CLASS, NUM_EXPERTS_ATTR = "Qwen3Moe", "Qwen3MoeExperts", "num_experts"


class HFQwen2MoePolicy(HFMoEPolicy):
    """`Qwen2MoeModel`, `Qwen2MoeForCausalLM` (the shared expert is a dense MLP and stays replicated)."""
    FAMILY, EXPERTS_CLASS, NUM_EXPERTS_ATTR = "Qwen2Moe", "Qwen2MoeExperts", "num_experts"


class HFDeepseekV3Policy(HFMoEPolicy):
    """`DeepseekV3Model`, `DeepseekV3ForCausalLM`: expert parallelism of the routed experts (`DeepseekV3NaiveMoe`); the
    router (group-limited top-k with correction bias), the shared experts and the multi-head latent attention are the
    model's own and stay replicated."""
    FAMILY, EXPERTS_CLASS, TP_ATTENTION, NUM_EXPERTS_ATTR = "DeepseekV3", "DeepseekV3NaiveMoe", False, "n_routed_experts"


class HFDeepseekV2Policy(HFMoEPolicy):
    """`DeepseekV2Model`, `DeepseekV2ForCausalLM` (expert parallelism only, like V3)."""
    FAMILY, EXPERTS_CLASS, TP_ATTENTION, NUM_EXPERTS_ATTR = "DeepseekV2", "DeepseekV2Experts", False, "n_routed_experts"
