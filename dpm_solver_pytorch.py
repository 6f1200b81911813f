"""Drop-in module name: `from dpm_solver_pytorch import NoiseScheduleVP, model_wrapper, DPM_Solver`
resolves to the H100-native implementation (dpm_solver_b200), so code written against the
reference's single-file library (README.md:227 of the reference) runs unchanged."""
from dpm_solver_b200 import (DPM_Solver, NoiseScheduleEDM, NoiseScheduleFlow, NoiseScheduleVP, UniPC,  # noqa: F401
                             expand_dims, interpolate_fn, model_wrapper)
