"""
tests/test_phi_cuda_facade.py once more, with the REAL engine (libphicuda.so) behind the facade: Fields of the `phi` test double in,
CUDA kernels in the middle, Fields out - on the GPU, with PhiML installed or copied into oracle/_ref.  Same test functions, same
assertions; only the `flow` fixture differs.
"""
import pytest
import torch

from _phiml import ensure_phiml

pytestmark = pytest.mark.gpu

if not torch.cuda.is_available():
    pytest.skip('needs a CUDA device', allow_module_level=True)
if not ensure_phiml():
    pytest.skip('PhiML not available (neither installed nor in oracle/_ref)', allow_module_level=True)

import test_phi_cuda_facade as cpu_tests  # noqa: E402
from test_phi_cuda_facade import (  # noqa: E402,F401
    test_import_exports_and_default_backend, test_make_incompressible_fields_in_fields_out, test_not_converged_is_raised_and_can_be_suppressed,
    test_ineligible_calls_fall_through_with_a_reason, test_centered_velocity_runs_the_wide_stencil_path, test_advection_wrappers,
    test_stencil_wrappers)

flow = cpu_tests.make_flow_fixture(real_engine=True)


def test_results_live_on_the_device(flow):
    import numpy as np
    from phiml import math
    from phiml.math import extrapolation as E
    v, _, _ = cpu_tests._velocity(flow, np.random.default_rng(0), E.PERIODIC)
    v2, p = flow.fluid.make_incompressible(v, (), flow.Solve('CG', 1e-5, 1e-5))
    assert p.values.native(p.values.shape).is_cuda
    assert v2.values[{'~vector': 'x'}].native(['b', 'x', 'y']).is_cuda
