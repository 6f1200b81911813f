"""Import the unmodified reference from oracle/_ref/*.pyc (built by oracle/build_ref.py).  TEST INFRASTRUCTURE:
only tests/, __graft_entry__.smoke() and bench.py's reference / cpu_baseline legs may use this; the product
package never imports it.

    ref = ref_loader.load("dpm_solver_pytorch")      # module with NoiseScheduleVP, model_wrapper, DPM_Solver

Falls back to the sources of the reference checkout (oracle/build_ref.py: $DPM_REFERENCE, default a `reference`
directory next to this repository or above it) when the bytecode has not been built yet. `available()` is the skip condition for tests.
"""
import importlib.machinery
import importlib.util
import os
import sys
import warnings

HERE = os.path.dirname(os.path.abspath(__file__))
REF_DIR = os.path.join(HERE, "_ref")
_cache = {}


def _source_path(name):
    from .build_ref import DEFAULT_REFERENCE as root, FILES
    p = os.path.join(root, FILES[name])
    return p if os.path.isfile(p) else None


def path(name):
    """File the module would be loaded from (pyc first), or None."""
    pyc = os.path.join(REF_DIR, name + ".pyc")
    if os.path.isfile(pyc):
        return pyc
    return _source_path(name)


def available(name="dpm_solver_pytorch"):
    return path(name) is not None


def spec(name, module_name=None):
    """importlib spec for a reference file, so that callers can register stub modules in sys.modules
    before `spec.loader.exec_module(mod)` (the example adapters import their model zoos at the top)."""
    p = path(name)
    if p is None:
        raise ImportError("reference file {!r} is neither in oracle/_ref (run oracle/build_ref.py) "
                          "nor in the reference checkout".format(name))
    module_name = module_name or "_dpm_ref_" + name
    if p.endswith(".pyc"):
        loader = importlib.machinery.SourcelessFileLoader(module_name, p)
        return importlib.util.spec_from_file_location(module_name, p, loader=loader)
    return importlib.util.spec_from_file_location(module_name, p)


def load(name="dpm_solver_pytorch", module_name=None, fresh=False):
    """Load (and cache) a reference module that needs no stubs."""
    key = (name, module_name)
    if not fresh and key in _cache:
        return _cache[key]
    s = spec(name, module_name)
    mod = importlib.util.module_from_spec(s)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", SyntaxWarning)
        s.loader.exec_module(mod)
    if module_name:
        sys.modules[module_name] = mod
    _cache[key] = mod
    return mod
