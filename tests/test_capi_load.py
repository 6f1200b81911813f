"""The C-ABI library loads without a GPU and exports every symbol include/dpm_solver_b200.h declares."""
import ctypes as C
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def declared_symbols():
    src = open(os.path.join(ROOT, "include", "dpm_solver_b200.h")).read()
    return sorted(set(re.findall(r"DPM_API\s+[\w\s\*]+?\b(dpm_\w+)\s*\(", src)))


def test_header_declares_the_expected_entry_points():
    syms = declared_symbols()
    for s in ("dpm_step", "dpm_solver_first_update", "dpm_multistep_second_update", "dpm_multistep_third_update",
              "dpm_singlestep_diff_update", "dpm_singlestep_third_taylor_update", "dpm_cfg_combine",
              "dpm_data_prediction", "dpm_dynamic_threshold", "dpm_lincomb", "dpm_version", "dpm_last_error"):
        assert s in syms


def test_library_exports_the_declared_symbols_and_version():
    """Every declared symbol is exported and bound, and dpm_version() is the header's DPM_B200_VERSION -- at least
    101, the first version whose dpm_adaptive_ctl carries beta_0_sq (a caller built against 100 leaves it unset)."""
    from dpm_solver_b200 import _lib
    from dpm_solver_b200.build import build
    build()
    handle = C.CDLL(str(_lib.LIB_PATH))
    for s in declared_symbols():
        assert hasattr(handle, s), s
    assert set(declared_symbols()) == set(_lib.PROTOTYPES)
    src = open(os.path.join(ROOT, "include", "dpm_solver_b200.h")).read()
    header_version = int(re.search(r"#define\s+DPM_B200_VERSION\s+(\d+)", src).group(1))
    L = _lib.lib()
    assert L.dpm_version() == header_version >= 101


def test_argument_validation_needs_no_gpu():
    from dpm_solver_b200 import _lib
    L = _lib.lib()
    assert L.dpm_step(None, None) == -1
    assert b"NULL" in L.dpm_last_error()
    d = _lib.StepDesc()
    d.n, d.form = 16, 5
    assert L.dpm_step(C.byref(d), None) == -1          # tensors missing
    d.state_dtype = 7
    assert L.dpm_step(C.byref(d), None) == -1          # bad dtype
    assert L.dpm_set_tuning(0, 96, 4) == 0 and L.dpm_set_tuning(2, 0, 0) == 0
    v, t, c = C.c_int(), C.c_int(), C.c_int()
    L.dpm_get_tuning(C.byref(v), C.byref(t), C.byref(c))
    assert (v.value, t.value, c.value) == (2, 0, 0)


def test_struct_layout_matches_header():
    """ctypes mirror of dpm_step_desc: 11 pointers, 2 u64, 8 i32, 12 floats, 1 pointer; and of dpm_adaptive_ctl."""
    from dpm_solver_b200 import _lib
    assert C.sizeof(_lib.StepDesc) == 11 * 8 + 2 * 8 + 8 * 4 + 12 * 4 + 8
    src = open(os.path.join(ROOT, "include", "dpm_solver_b200.h")).read()
    body = src[src.index("typedef struct dpm_step_desc {"):src.index("} dpm_step_desc;")]
    names = re.findall(r"\b(\w+)\s*(?:,|;)", re.sub(r"/\*.*?\*/", "", body, flags=re.S))
    assert [n for n, _ in _lib.StepDesc._fields_] == names
    body = src[src.index("typedef struct dpm_adaptive_ctl {"):src.index("} dpm_adaptive_ctl;")]
    names = re.findall(r"\b(\w+)\s*(?:,|;)", re.sub(r"/\*.*?\*/", "", body, flags=re.S))
    assert [n for n, _ in _lib.AdaptiveCtl._fields_] == names


def test_cpu_tensors_are_refused():
    import torch
    from dpm_solver_b200 import ops
    be = ops.CudaBackend()
    with pytest.raises(RuntimeError, match="CUDA-only"):
        be.step(ops.StepArgs(form=1, x=torch.zeros(8), m0=torch.zeros(8), a=1.0, c0=1.0))


def test_header_is_plain_c_and_links(tmp_path):
    """include/dpm_solver_b200.h compiles as C99 (-pedantic) and a C program links against the library and calls
    it without a GPU: the boundary really is a C-ABI, not a C++ or torch interface."""
    import shutil
    import subprocess
    from dpm_solver_b200 import _lib
    if shutil.which("gcc") is None:
        pytest.skip("gcc not available")
    src = tmp_path / "client.c"
    src.write_text(r"""
#include <stdio.h>
#include <string.h>
#include "dpm_solver_b200.h"
int main(void) {
  dpm_step_desc d;
  memset(&d, 0, sizeof d);
  if (dpm_version() != DPM_B200_VERSION) return 1;
  if (dpm_step(NULL, NULL) != DPM_ERR_ARG || strstr(dpm_last_error(), "NULL") == NULL) return 2;
  if (dpm_step(&d, NULL) != DPM_OK) return 3;             /* n == 0: nothing to do */
  d.n = 16; d.form = DPM_FORM_MS3;
  if (dpm_step(&d, NULL) != DPM_ERR_ARG) return 4;         /* tensors missing */
  printf("%zu\n", sizeof d);
  return 0;
}
""")
    exe = tmp_path / "client"
    libdir = str(_lib.LIB_PATH.parent) if hasattr(_lib.LIB_PATH, "parent") else os.path.dirname(str(_lib.LIB_PATH))
    subprocess.run(["gcc", "-std=c99", "-Wall", "-Wextra", "-Werror", "-pedantic", "-I", os.path.join(ROOT, "include"), str(src),
                    "-L", libdir, "-ldpmsolver_b200", "-Wl,-rpath," + libdir, "-o", str(exe)], check=True)
    r = subprocess.run([str(exe)], capture_output=True, text=True)
    assert r.returncode == 0, (r.returncode, r.stdout, r.stderr)
    assert int(r.stdout.strip()) == C.sizeof(_lib.StepDesc)
