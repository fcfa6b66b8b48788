import pytest


def test_build_compiles_all_native_libraries():
    import __graft_entry__ as g

    g.build()


@pytest.mark.gpu
def test_smoke_runs_native_kernels():
    import __graft_entry__ as g

    g.smoke()


def test_extension_registry():
    """Every reference extension name resolves to an in-tree sm_90a library descriptor (reference: extensions/)."""
    from colossalai_b200.extensions import ALL_EXTENSIONS, CppExtension, CudaExtension, get_extension

    for name in ("cpu_adam_x86", "fused_optim_cuda", "layernorm_cuda", "moe_cuda", "scaled_masked_softmax_cuda",
                 "scaled_upper_triangle_masked_softmax_cuda", "inference_ops_cuda"):
        assert name in ALL_EXTENSIONS and ALL_EXTENSIONS[name].is_available()
    assert isinstance(get_extension("cpu_adam_x86"), CppExtension)
    assert isinstance(get_extension("gemm_tcgen05"), CudaExtension)
    assert get_extension("cpu_adam_x86").build_aot().exists()
