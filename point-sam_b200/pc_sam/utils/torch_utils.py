"""/root/reference/pc_sam/utils/torch_utils.py:28-38."""
from torch import nn


def replace_with_fused_layernorm(module: nn.Module):
    """No-op: every LayerNorm of this implementation already runs in the fused sm_90a kernels
    (psam_layernorm_f32 and the LN-fused epilogues); module types and state-dict keys are unchanged,
    exactly as after apex's swap."""
    return module
