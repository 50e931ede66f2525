"""vampnet.modules.activations (reference vampnet/modules/activations.py).  On the generation path GatedGELU is the
epilogue of the FFN up-projection GEMM (vampnet_b200/csrc/gemm_wgmma.cu) and Snake the epilogue of the codec
convolutions; there are no standalone activation modules to export.  get_activation answers by name so that code
which only *asks* for an activation class fails with a clear message instead of an ImportError."""


def get_activation(name: str = "relu"):
    """activations.py:44-54."""
    if name in ("relu", "gelu", "geglu", "snake"):
        raise NotImplementedError(
            f"activation '{name}' is fused into the sm_90a kernels (GEGLU: FFN-up GEMM epilogue; snake: codec conv "
            "epilogue) and has no standalone module in this build")
    raise ValueError(f"Unrecognized activation {name}")
