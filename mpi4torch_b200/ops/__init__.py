"""Functional ops on top of the communicator: fused-epilogue collectives and
the Allreduce->GEMM fused linear layer, the data-parallel two-layer MLP."""
from .functional import allreduce, allreduce_mean, allreduce_sgd_step_, average_parameters_flat
from .fused_linear import (AccumulatedSGD, InBackwardSGD, allreduce_linear, dp_linear_mse, dp_linear_mse_supported,
                           has_fused_kernel, in_backward_sgd_supported)
from .expert_mlp import (expert_group_starts, expert_mlp, expert_mlp_supported, grouped_expert_mlp,
                         grouped_expert_mlp_supported)
from .fp8 import dp_linear_mse_fp8_supported
from .fused_mlp import (dp_mlp_cross_entropy, dp_mlp_cross_entropy_supported, dp_mlp_mse, dp_mlp_mse_supported,
                        mlp_in_backward_sgd_supported)

__all__ = ["allreduce", "allreduce_mean", "allreduce_sgd_step_", "average_parameters_flat", "allreduce_linear",
           "has_fused_kernel", "dp_linear_mse", "dp_linear_mse_supported", "InBackwardSGD", "in_backward_sgd_supported",
           "dp_mlp_mse", "dp_mlp_mse_supported", "mlp_in_backward_sgd_supported", "dp_mlp_cross_entropy",
           "dp_mlp_cross_entropy_supported", "AccumulatedSGD", "dp_linear_mse_fp8_supported", "expert_mlp",
           "expert_mlp_supported", "expert_group_starts", "grouped_expert_mlp", "grouped_expert_mlp_supported"]
