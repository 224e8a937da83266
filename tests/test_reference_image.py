"""etxb_reference_image_file_read (Open Reference Image): the float4 pixels the image pool keeps of a file, on files the module writes and, where the
reference tree is built, byte for byte against the reference's own ImagePool (oracle/ref_image_pool.cxx).  CPU only."""
import warnings

import numpy as np
import pytest

from etx_tracer_b200 import api

f32 = np.float32


def _pool_8bit(u8):
    """ImagePool's 8-bit path as restated in numpy: sRGB -> linear on RGB, to_ubyte4 truncation, then the UNORM read (/255)."""
    f = u8.astype(f32) / f32(255)
    lin = f.copy()
    rgb = f[..., :3]
    lin[..., :3] = np.where(rgb <= f32(0.04045), rgb / f32(12.92), (((rgb.astype(np.float64) + 0.055) / 1.055) ** 2.4).astype(f32))
    return (np.clip(lin, 0, 1) * f32(255)).astype(np.uint8).astype(f32) / f32(255)


def test_film_written_as_exr_reads_back_identical(tmp_path):
    rng = np.random.default_rng(3)
    film = (rng.uniform(0, 8, (24, 40, 4)) ** 2).astype(f32)
    api.write_exr(str(tmp_path / "film.exr"), film)
    back = api.read_reference_image(str(tmp_path / "film.exr"))
    assert back.shape == film.shape and np.array_equal(back.view(np.uint32), film.view(np.uint32))


def test_exr_non_finite_and_negative_values_are_cleaned_as_the_pool_does(tmp_path):
    img = np.ones((4, 4, 4), f32)
    img[0, 0] = [np.inf, -np.inf, np.nan, -2.0]
    img[1, 1] = [0.5, -0.0, 70000.0, 1.0]
    api.write_exr(str(tmp_path / "odd.exr"), img)
    back = api.read_reference_image(str(tmp_path / "odd.exr"))
    assert np.array_equal(back[0, 0], [65504.0, 65504.0, 0.0, 0.0])  # either infinity -> 65504, NaN and negatives -> 0
    assert np.array_equal(back[1, 1], f32([0.5, 0.0, 70000.0, 1.0]))
    assert np.array_equal(back[2:], img[2:])


def test_8bit_png_goes_through_srgb_to_linear_and_truncation(tmp_path):
    v = np.arange(256, dtype=np.uint8).reshape(16, 16)
    rgba = np.stack([v, v[::-1], v.T, v], axis=-1)
    api.write_png(str(tmp_path / "ramp.png"), rgba)
    back = api.read_reference_image(str(tmp_path / "ramp.png"))
    want = _pool_8bit(rgba)
    assert back.shape == (16, 16, 4)
    assert np.array_equal(back[..., 3], rgba[..., 3].astype(f32) / f32(255))  # alpha: no curve, the byte read back
    # powf against float64 numpy may move a value across a truncation step
    assert np.abs(back - want).max() <= 1.0 / 255 + 1e-7 and (back == want).mean() > 0.99


def test_unreadable_file_is_the_white_placeholder_with_a_warning(tmp_path):
    (tmp_path / "bad.png").write_bytes(b"not an image")
    with pytest.warns(UserWarning, match="placeholder"):
        back = api.read_reference_image(str(tmp_path / "bad.png"))
    assert back.shape == (1, 1, 4) and np.array_equal(back, np.ones((1, 1, 4), f32))
    with pytest.warns(UserWarning):
        assert api.read_reference_image(str(tmp_path / "missing.exr")).shape == (1, 1, 4)


def _write_pfm(path, rgb, grey=False):
    """The reference's PFM variant (image_pool.cxx:463-541): 'PF' / 'Pf', width, height and scale on lines of their own, then the floats."""
    h, w = rgb.shape[:2]
    with open(path, "wb") as f:
        f.write(b"Pf\n" if grey else b"PF\n")
        f.write(f"{w}\n{h}\n-1.0\n".encode())
        f.write(np.ascontiguousarray(rgb, "<f4").tobytes())


def _write_hdr(path, rgbe):
    """Radiance RGBE, flat scan lines (a width under 8 is never run-length encoded)."""
    h, w = rgbe.shape[:2]
    with open(path, "wb") as f:
        f.write(f"#?RADIANCE\nFORMAT=32-bit_rle_rgbe\n\n-Y {h} +X {w}\n".encode())
        f.write(np.ascontiguousarray(rgbe, np.uint8).tobytes())


def test_hdr_and_pfm_pixels_come_back_as_read(tmp_path):
    """ImagePool cleans float pixels in its OpenEXR branch only: HDR and PFM keep negatives, NaN and inf."""
    rgb = np.array([[[-1.5, np.nan, np.inf], [0.25, -0.0, 3.0]]], np.float32)
    _write_pfm(tmp_path / "odd.pfm", rgb)
    back = api.read_reference_image(str(tmp_path / "odd.pfm"))
    assert back.shape == (1, 2, 4) and np.array_equal(back[..., 3], np.ones((1, 2), f32))
    assert np.array_equal(back[..., :3].view(np.uint32), rgb.view(np.uint32))
    _write_pfm(tmp_path / "grey.pfm", np.array([[-2.0, 0.5]], np.float32), grey=True)
    assert np.array_equal(api.read_reference_image(str(tmp_path / "grey.pfm"))[0], f32([[-2, -2, -2, 1], [0.5, 0.5, 0.5, 1]]))
    rgbe = np.array([[[128, 64, 32, 129], [0, 0, 0, 0], [255, 255, 255, 200]]], np.uint8)
    _write_hdr(tmp_path / "flat.hdr", rgbe)
    back = api.read_reference_image(str(tmp_path / "flat.hdr"))
    assert back.shape == (1, 3, 4) and back[0, 0, 0] == 1.0 and np.array_equal(back[0, 1], f32([0, 0, 0, 1]))


# ---- against the reference's own ImagePool (oracle/ref_image_pool.cxx over libreference_loader.so), where it is built --------------------------
def _refpool():
    import ctypes as C
    import os
    path = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle", "_ref", "libreference_image_pool.so")
    if not os.path.exists(path):
        pytest.skip("oracle/_ref/libreference_image_pool.so not present (built where the reference tree exists)")
    lib = C.CDLL(path)
    lib.refpool_read.argtypes = [C.c_char_p, C.POINTER(C.c_uint32), C.POINTER(C.c_uint32), C.c_void_p, C.c_uint64]

    def read(file_name):
        w, h = C.c_uint32(0), C.c_uint32(0)
        lib.refpool_read(os.fsencode(file_name), C.byref(w), C.byref(h), None, 0)
        out = np.zeros((h.value, w.value, 4), np.float32)
        assert lib.refpool_read(os.fsencode(file_name), C.byref(w), C.byref(h), out.ctypes.data_as(C.c_void_p), out.nbytes) == 0
        return out

    return read


def _files(tmp_path):
    """Every kind of file the viewer's Open Reference Image takes, including values the pool has to clean or keep."""
    rng = np.random.default_rng(5)
    made = {}
    Image = pytest.importorskip("PIL.Image")
    rgba = rng.integers(0, 256, (9, 13, 4), dtype=np.uint8)
    for mode, name, arr in (("RGBA", "rgba.png", rgba), ("RGB", "rgb.png", rgba[..., :3]), ("L", "grey.png", rgba[..., 0])):
        Image.fromarray(np.ascontiguousarray(arr), mode).save(tmp_path / name)
        made[name] = tmp_path / name
    Image.fromarray(np.ascontiguousarray(rgba[..., :3]), "RGB").save(tmp_path / "photo.jpg", quality=90)
    made["photo.jpg"] = tmp_path / "photo.jpg"
    exr = (rng.uniform(0, 4, (7, 5, 4))).astype(np.float32)
    exr[0, 0] = [np.inf, -np.inf, np.nan, -2.0]
    exr[3, 2] = [-0.0, 70000.0, 1e-30, 0.5]
    api.write_exr(str(tmp_path / "odd.exr"), exr)
    made["odd.exr"] = tmp_path / "odd.exr"
    rgbe = rng.integers(0, 256, (3, 5, 4), dtype=np.uint8)
    rgbe[0, 0] = 0
    _write_hdr(tmp_path / "flat.hdr", rgbe)
    made["flat.hdr"] = tmp_path / "flat.hdr"
    pfm = rng.normal(0, 2, (4, 6, 3)).astype(np.float32)
    pfm[1, 1] = [np.nan, np.inf, -np.inf]
    _write_pfm(tmp_path / "odd.pfm", pfm)
    made["odd.pfm"] = tmp_path / "odd.pfm"
    (tmp_path / "bad.png").write_bytes(b"not an image")
    made["bad.png"] = tmp_path / "bad.png"
    made["missing.exr"] = tmp_path / "missing.exr"
    return made


def test_reader_equals_the_reference_image_pool_byte_for_byte(tmp_path):
    ref_read = _refpool()
    for name, path in _files(tmp_path).items():
        want = ref_read(path)
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")  # the placeholder's warning
            got = api.read_reference_image(str(path))
        assert got.shape == want.shape and np.array_equal(got.view(np.uint32), want.view(np.uint32)), name
