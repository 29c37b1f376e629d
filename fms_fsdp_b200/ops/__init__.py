from fms_fsdp_b200.ops.functional import (  # noqa: F401
    add_rmsnorm, attention, causal_conv1d, cross_entropy, cross_entropy_z, document_segments, embedding, gated_mlp,
    get_kernel_path, kernels_for, linear, linear_cross_entropy, linear_cross_entropy_z, moe_mlp, qkv_attention,
    rmsnorm, rmsnorm_fork, rmsnorm_gated, rope_, selective_scan, set_kernel_path, ssd_scan, swiglu,
)
