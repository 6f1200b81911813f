"""Drop-in module name: `from dpm_solver_pytorch import NoiseScheduleVP, model_wrapper, DPM_Solver`
resolves to the H100-native implementation (dpm_solver_b200), so code written against the
reference's single-file library (README.md:227 of the reference) runs unchanged."""
from dpm_solver_b200 import (DPM_Solver, NoiseScheduleFlow, NoiseScheduleVP, UniPC, expand_dims,  # noqa: F401
                             interpolate_fn, model_wrapper)
