"""dpm_solver_b200 -- H100-native (sm_90a) implementation of DPM-Solver's per-step update path.

Drop-in for the three public names of LuChengTHU/dpm-solver's `dpm_solver_pytorch.py`:

    from dpm_solver_b200 import NoiseScheduleVP, model_wrapper, DPM_Solver

plus `NoiseScheduleFlow` and `model_type="flow"` for flow-matching (rectified-flow) models, `NoiseScheduleEDM` and
`model_type="edm"` for EDM-preconditioned models, and the UniPC multistep sampler `UniPC` (unipc.py).

The arithmetic runs in hand-written CUDA kernels behind a C-ABI shared library
(include/dpm_solver_b200.h, built by `python -m dpm_solver_b200.build`). There is no CPU or
PyTorch fallback: CUDA tensors only, and a missing library raises.
"""
from .schedule import NoiseScheduleEDM, NoiseScheduleFlow, NoiseScheduleVP, expand_dims, interpolate_fn
from .diffedit import DiffEditCorrector
from .solver import DPM_Solver, WrappedModel, model_wrapper
from .unipc import UniPC

__version__ = "0.1.0"
__all__ = ["NoiseScheduleVP", "NoiseScheduleFlow", "NoiseScheduleEDM", "model_wrapper", "DPM_Solver", "UniPC", "WrappedModel", "interpolate_fn",
           "expand_dims", "DiffEditCorrector"]
