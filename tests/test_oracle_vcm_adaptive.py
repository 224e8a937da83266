"""The oracle's VCM CameraAdaptive layer (oracle/oracle_vcm_adaptive.cxx): film.cxx's every-other-sample mean, which the reference's Film keeps
for CPUVCM as for the path tracer and which the device's VCM keeps for the denoiser (DESIGN §13).  Runs without a GPU."""
import numpy as np
import pytest

from conftest import bit_equal
from etx_tracer_b200 import scenes, structs as S


@pytest.fixture(scope="module")
def adaptive_oracle():
    from oracle import oracle_vcm_adaptive_py
    if not oracle_vcm_adaptive_py.available():
        pytest.skip("oracle/_ref/liboracle_vcm_adaptive_parity.so not built (run build() where /root/reference exists)")
    return oracle_vcm_adaptive_py


def _scene(spectral):
    return scenes.cornell_box(24, 20, samples=64, spectral=spectral, sphere=spectral, sphere_segments=16, sphere_rings=9)


def _run(mod, sd, size, first, iterations):
    o = mod.Oracle(sd)
    o.set_film_pixel_size(size)
    o.begin(first)
    o.run(iterations)
    return o


def _lerp32(a, b, t):
    """lerp (math.hxx:691) in float32, no contraction"""
    t = np.float32(t)
    return a * (np.float32(1.0) - t) + b * t


@pytest.mark.parametrize("spectral", [False, True])
@pytest.mark.parametrize("size", [1, 2, 3])
def test_one_iteration_leaves_the_camera_layer(adaptive_oracle, spectral, size):
    o = _run(adaptive_oracle, _scene(spectral), size, 0, 1)
    cam = o.film(S.FILM_CAMERA)[..., :3]
    assert cam.any() and bit_equal(o.film(S.FILM_CAMERA_ADAPTIVE)[..., :3], cam)


@pytest.mark.parametrize("spectral", [False, True])
@pytest.mark.parametrize("size", [1, 2, 3])
def test_the_layer_follows_the_even_sample_rule(adaptive_oracle, spectral, size):
    """VCM iterations are independent (the index sets the seeds and the radius): a one-iteration run begun at k holds iteration k's camera
    values, and after K iterations the layer is the running lerp over the even ones"""
    sd = _scene(spectral)
    K = 5
    values = [_run(adaptive_oracle, sd, size, k, 1).film(S.FILM_CAMERA)[..., :3] for k in range(K)]
    o = _run(adaptive_oracle, sd, size, 0, K)
    want = values[0]
    for k in range(2, K, 2):
        want = _lerp32(values[k], want, np.float64(k) / (k + 2.0))
    adaptive = o.film(S.FILM_CAMERA_ADAPTIVE)[..., :3]
    assert bit_equal(adaptive, want)
    assert not bit_equal(adaptive, o.film(S.FILM_CAMERA)[..., :3])


def test_everything_else_is_the_preview_oracle(adaptive_oracle):
    """the layer is all the library adds: the camera and light layers, and the path tracer's layers, are the preview oracle's"""
    from oracle import oracle_preview_py
    if not oracle_preview_py.available():
        pytest.skip("oracle/_ref/liboracle_preview_parity.so not built")
    sd = _scene(True)
    for pt in (False, True):
        a, b = adaptive_oracle.Oracle(sd), oracle_preview_py.Oracle(sd)
        for o in (a, b):
            if pt:
                o.set_integrator(S.INTEGRATOR_PT)
                o.pt_set_options(S.default_pt_options())
            o.set_film_pixel_size(2)
            o.begin(0)
            o.run(3)
        layers = (S.FILM_CAMERA, S.FILM_LIGHT) + ((S.FILM_NORMALS, S.FILM_ALBEDO, S.FILM_CAMERA_ADAPTIVE) if pt else ())
        for layer in layers:
            assert bit_equal(a.film(layer)[..., :3], b.film(layer)[..., :3]), (pt, layer)
