"""CPU tests of the orthographic kernels (build.py ORTHO_SOURCES) in the emulator (tests/emu/ortho.py).  The case matrix that launches
every orthographic kernel, on ordinary and on hostile depth (tests/hostile_cases.py) under extreme cameras and tolerances, is
tests/unit_matrix.py's, run by test_unit_matrix_emulated.py."""
import numpy as np

import unit_matrix as um
from emu import ortho
from ortho_oracle import OrthoOracle


def test_matrix_names_every_kernel_built():
    assert set().union(*(um.expected_kernels(c) for c in um.CASES if c.unit == "ortho")) == ortho.kernels()


def test_emulator_units_match_libmeao_tables():
    assert ortho.kernel_units() == {"prepare_depth_ortho.cu": 12, "prepare_depth_ortho_layered.cu": 12, "prepare_depth_array_ortho.cu": 4,
                                    "render_ao_ortho.cu": 12, "render_ao_ortho_layered.cu": 12, "blur_upsample_lin_ortho.cu": 12}


# ---- extreme cameras ------------------------------------------------------------------------------------------------------------
def test_it_overflows_camera_reaches_inf():
    """The camera of the matrix's it_overflows cases (tests/unit_matrix.py) does send it_i of the coarse levels to inf."""
    W, H = um.HOSTILE_FED
    cam = um.hostile_camera("it_overflows", W, H, True, orthographic=True)
    orc = OrthoOracle(W, H, near=cam.nearClipPlane, far=cam.farClipPlane, tan_half_fov_h_=1.0 / cam.projection00)
    assert np.isinf(orc.inv_thickness(4)).any()
