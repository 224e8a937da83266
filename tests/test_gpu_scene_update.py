"""etxb_update_scene / etxb_group_update_scene: a context restarted on an edited scene renders what a fresh context renders after
etxb_upload_scene of the same PODs, while the device keeps what the edit did not change.  Context A uploads S, renders 2 iterations,
updates to S' and renders 3 more; context B uploads S' and renders 3.  The GPU tests run with -m gpu; the adapter tests at the end run
without a device."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from conftest import ROOT, bit_equal, rel_l2
from etx_tracer_b200 import build as etx_build, scenes, structs as S

gpu = pytest.mark.gpu
C1 = dict(samples=16, spectral=False)


# ---- edited scenes: every pair is built by the scenes.py generators, the geometry is identical unless the edit says otherwise -----------
def _cornell(edit=None, width=32, height=32, **kw):
    args = dict(C1, **kw)
    sd = scenes.cornell_box(width, height, samples=args["samples"], spectral=args["spectral"], finalize=False)
    if edit:
        edit(sd)
    return sd.finalize(samples=args["samples"], spectral=args["spectral"])


def _move_camera(sd):
    sd.set_camera([0.2, 1.1, 3.6], [0.0, 0.9, -6.18], [0.0, 1.0, 0.0], sd.width, sd.height, 39.597755335771296, clip_near=0.1, clip_far=100.0)


def _plastic_box(lambert=False, roughness=None, width=32, height=32):
    """material_box("plastic"); lambert=True gives its "test" material the white wall's Lambert record (same geometry, same material count)"""
    sd = scenes.material_box("plastic", width, height, samples=16)
    test, white = sd.material_names["test"], sd.material_names["white"]
    if lambert:
        sd.a_materials[test] = sd.a_materials[white]
    if roughness is not None:
        sd.a_materials[test]["roughness"]["value"][:2] = roughness
    return sd


def _scale_spectrum(sd, index, k):
    sd.a_spectra[index]["entries"]["power"] *= np.float32(k)
    sd.a_spectra[index]["integrated"] *= np.float32(k)


def _reflectance_edit():
    s1 = _cornell()
    s2 = _cornell()
    _scale_spectrum(s2, int(s2.a_materials[s2.material_names["leftWall"]]["reflectance"]["spectrum_index"]), 0.6)
    return s1, s2


def _emission(sd):
    sd.materials[sd.material_names["light"]]["emission"]["spectrum_index"] = sd.add_spectrum(scenes.spd_rgb_luminance([4.0, 9.0, 2.5]))


def _emissive_wall(sd):
    sd.materials[sd.material_names["rightWall"]]["emission"]["spectrum_index"] = sd.add_spectrum(scenes.spd_rgb_luminance([0.6, 0.9, 0.3]))


def _camera_medium(sd):
    sd.camera["medium_index"] = sd.add_medium(absorption=(0.05, 0.05, 0.05), scattering=(0.3, 0.3, 0.35))


def _opacity(sd):
    sd.materials[sd.material_names["grey"]]["opacity"] = 0.5


def _move_vertex(sd):
    sd.vertices[-1]["pos"][-1] += np.float32(0.05)  # a corner of the short box


def _cloud(absorption=1.0, density=1.0):
    sd = scenes.media_box("cloud")
    m = sd.a_mediums[0]
    if absorption != 1.0:
        _scale_spectrum(sd, int(m["absorption_index"]), absorption)
    if density != 1.0:
        grid = np.frombuffer((C.c_float * int(m["density"]["count"])).from_address(int(m["density"]["a"])), dtype=np.float32)
        grid[: grid.size // 3] *= np.float32(density)
    return sd


def _env_image(sd):
    return int(sd.a_profiles[sd.a_profiles["cls"] == S.EMITTER_ENVIRONMENT]["emission"]["image_index"][0])


def _sky(pixel_edit=False):
    sd = scenes.sky_room(32, 32)
    if pixel_edit:
        im = sd.a_images[_env_image(sd)]
        px = np.frombuffer((C.c_float * 4).from_address(int(im["pixels"]["a"])), dtype=np.float32)
        px[:3] *= np.float32(1.5)
    return sd


EDITS = {
    "camera_moved": lambda: (_cornell(), _cornell(_move_camera)),
    "film_larger": lambda: (_cornell(), _cornell(width=48, height=40)),
    "film_smaller": lambda: (_cornell(width=48, height=40), _cornell()),
    "plastic_roughness": lambda: (_plastic_box(), _plastic_box(roughness=0.3)),
    "reflectance_spectrum": _reflectance_edit,
    "lambert_to_plastic": lambda: (_plastic_box(lambert=True), _plastic_box()),
    "plastic_to_lambert": lambda: (_plastic_box(), _plastic_box(lambert=True)),
    "emission_colour": lambda: (_cornell(), _cornell(_emission)),
    "wall_emissive": lambda: (_cornell(), _cornell(_emissive_wall)),
    "medium_absorption": lambda: (_cloud(), _cloud(absorption=2.0)),
    "density_grid": lambda: (_cloud(), _cloud(density=0.5)),
    "camera_medium": lambda: (_cornell(), _cornell(_camera_medium)),
    "env_pixel": lambda: (_sky(), _sky(pixel_edit=True)),
    "rgb_to_spectral": lambda: (_cornell(), _cornell(spectral=True)),
    "spectral_to_rgb": lambda: (_cornell(spectral=True), _cornell()),
    "opacity": lambda: (_cornell(), _cornell(_opacity)),
    "vertex_moved": lambda: (_cornell(), _cornell(_move_vertex)),
}

VCM_BUFFERS = ((S.BUF_LIGHT_SAMPLER, np.uint32), (S.BUF_CAMERA_SAMPLER, np.uint32), (S.BUF_LIGHT_PATH_COUNT, np.uint32), (S.BUF_LIGHT_PATH_OFFSET, np.uint32),
               (S.BUF_LV_POS, np.float32), (S.BUF_LV_THROUGHPUT, np.float32), (S.BUF_LV_MIS, np.float32))
PT_LAYERS = (S.FILM_CAMERA, S.FILM_NORMALS, S.FILM_ALBEDO, S.FILM_CAMERA_ADAPTIVE)
PT_BUFFERS = ((S.BUF_PIXEL_INFO, np.uint32), (S.BUF_PIXEL_ERROR, np.float32))


@pytest.fixture(scope="module")
def api():
    from etx_tracer_b200 import api as m
    return m


def _iterate(g, n):
    for _ in range(n):
        g.iterate()
    g.wait()


def _updated(api, cls, s1, s2, flavor):
    """context A: S, 2 iterations, update to S', 3 iterations (no run(): the update itself arms iteration 0)"""
    a = cls(s1, flavor=flavor)
    a.render(2)
    info = a.update_scene(s2)
    _iterate(a, 3)
    return a, info


def _fresh(api, cls, s2, flavor):
    b = cls(s2, flavor=flavor)
    b.render(3)
    return b


def _vcm_state(g):
    out = {f"buf{bid}": g.buffer(bid, dt) for bid, dt in VCM_BUFFERS}
    out["film_camera"] = g.film(S.FILM_CAMERA)[..., :3]
    out["film_light"] = g.film(S.FILM_LIGHT)[..., :3]
    return out


def _pt_state(g):
    out = {f"layer{k}": g.film(k)[..., :3] for k in PT_LAYERS}
    out.update({f"buf{bid}": g.buffer(bid, dt) for bid, dt in PT_BUFFERS})
    return out


@gpu
@pytest.mark.parametrize("edit", sorted(EDITS))
def test_parity_vcm_update_equals_fresh_upload(api, edit):
    s1, s2 = EDITS[edit]()
    a, info = _updated(api, api.GPUVCM, s1, s2, "parity")
    b = _fresh(api, api.GPUVCM, s2, "parity")
    sa, sb = _vcm_state(a), _vcm_state(b)
    for key in sa:
        if key == "film_light":
            assert rel_l2(sa[key], sb[key]) < 1e-6, key  # float-atomic splats
        else:
            assert bit_equal(sa[key], sb[key]), key
    assert bool(info["kept"] & S.KEPT_GEOMETRY) == (edit != "vertex_moved")
    if edit in ("camera_moved", "plastic_roughness", "reflectance_spectrum", "emission_colour", "medium_absorption", "density_grid", "env_pixel"):
        assert info["kept"] & S.KEPT_PATH_STATE
    if edit in ("film_larger", "film_smaller", "lambert_to_plastic"):
        assert not info["kept"] & S.KEPT_PATH_STATE
    if edit == "env_pixel":
        assert info["images_uploaded"] == 1 and info["images_kept"] == int(s2.scene["images"]["count"][0]) - 1
    if edit == "density_grid":
        assert (info["grids_uploaded"], info["grids_kept"]) == (1, 0)
    if edit == "medium_absorption":
        assert (info["grids_uploaded"], info["grids_kept"]) == (0, 1)
    a.close()
    b.close()


@gpu
@pytest.mark.parametrize("edit", sorted(EDITS))
def test_parity_path_tracer_update_equals_fresh_upload(api, edit):
    s1, s2 = EDITS[edit]()
    a, _ = _updated(api, api.GPUPathTracing, s1, s2, "parity")
    b = _fresh(api, api.GPUPathTracing, s2, "parity")
    sa, sb = _pt_state(a), _pt_state(b)
    for key in sa:
        assert bit_equal(sa[key], sb[key]), key
    a.close()
    b.close()


# product-build outputs that are float-atomic sums: the light image (splats land in any order), the camera film (in scenes with a
# connection stage, the vertex connections of one path add into its accumulator with atomics, kernels.cuh k_camera_connect /
# k_shadow_resolve) and every film made of them
FLOAT_ATOMIC = ("film_light", "film_camera", "film_result")


def _within_fresh_spread(a, b1, b2, key):
    """product build: a float-atomic sum is compared with the 1e-6 relative-L2 bound, whatever the two fresh contexts show (their order differs
    from run to run, so they may agree by chance); every other output (sampler states, light-path counts and offsets, light-vertex pool) is
    deterministic, so the two fresh contexts agree on it bit for bit and A matches them bit for bit"""
    if key in FLOAT_ATOMIC:
        assert rel_l2(a, b1) <= 1e-6, (key, rel_l2(a, b1), rel_l2(b2, b1))
    else:
        assert bit_equal(b1, b2), f"{key}: two fresh contexts differ"
        assert bit_equal(a, b1), key


@gpu
@pytest.mark.parametrize("edit", sorted(EDITS))
def test_product_build_update_equals_fresh_upload(api, edit):
    s1, s2 = EDITS[edit]()
    b1, b2 = _fresh(api, api.GPUVCM, s2, "fast"), _fresh(api, api.GPUVCM, s2, "fast")
    a, info = _updated(api, api.GPUVCM, s1, s2, "fast")
    s1_, s2_, sa = _vcm_state(b1), _vcm_state(b2), _vcm_state(a)
    for key in sa:
        _within_fresh_spread(sa[key], s1_[key], s2_[key], key)
    assert a.debug_select_tree(True) == b1.debug_select_tree(True)  # the 4-wide tree exists exactly when a fresh upload builds one
    if edit == "lambert_to_plastic":
        assert info["kept"] & S.KEPT_GEOMETRY and not info["kept"] & S.KEPT_WIDE_TREE and info["bvh_seconds"] > 0.0
        assert a.debug_select_tree(True)
    if edit == "plastic_to_lambert":
        assert info["kept"] & S.KEPT_GEOMETRY and not a.debug_select_tree(True)
    if edit == "plastic_roughness":
        assert info["kept"] & S.KEPT_WIDE_TREE and info["bvh_seconds"] == 0.0
    for g in (a, b1, b2):
        g.close()


@gpu
@pytest.mark.parametrize("make", [lambda: (_plastic_box(), _plastic_box()), lambda: (_sky(), _sky()), lambda: (_cloud(), _cloud())], ids=["plastic", "sky", "cloud"])
def test_camera_only_update_keeps_everything(api, make):
    s1, s2 = make()
    _move_camera(s2)
    a = api.GPUVCM(s1, flavor="fast")
    a.render(1)
    wide = a.debug_select_tree(True)
    info = a.update_scene(s2)
    expect = S.KEPT_GEOMETRY | S.KEPT_PATH_STATE | (S.KEPT_WIDE_TREE if wide else 0)
    assert info["kept"] == expect, info
    assert info["bvh_seconds"] == 0.0 and info["images_uploaded"] == 0 and info["grids_uploaded"] == 0
    assert info["images_kept"] == int(s2.scene["images"]["count"][0]) and info["grids_kept"] == int((s2.a_mediums["cls"] == 1).sum())
    assert info["fingerprint_seconds"] > 0.0 and info["total_seconds"] >= info["fingerprint_seconds"]
    geometry = int(s2.scene["vertices"]["count"][0]) * S.VERTEX.itemsize + int(s2.scene["triangles"]["count"][0]) * S.TRIANGLE.itemsize
    pixels = sum(int(im["isize"][0]) * int(im["isize"][1]) * (16 if int(im["format"]) == 1 else 4) for im in s2.a_images)
    grids = sum(int(m["density"]["count"]) * 4 for m in s2.a_mediums if int(m["cls"]) == 1)
    assert info["bytes_hashed"] >= geometry + pixels + grids
    assert a.debug_select_tree(True) == wide
    a.close()


@gpu
def test_refused_update_leaves_the_previous_scene(api):
    s1 = _cornell()
    bad = _cornell()
    bad.a_materials[bad.material_names["grey"]]["reflectance"]["image_index"] = 99
    a = api.GPUVCM(s1, flavor="parity")
    a.render(2)
    with pytest.raises(api.EtxbError) as e:
        a.update_scene(bad)
    assert e.value.code == -1 and "image index" in str(e.value)
    a.render(3)
    b = _fresh(api, api.GPUVCM, s1, "parity")
    sa, sb = _vcm_state(a), _vcm_state(b)
    for key in sa:
        assert (rel_l2(sa[key], sb[key]) < 1e-6) if key == "film_light" else bit_equal(sa[key], sb[key]), key
    a.close()
    b.close()


@gpu
def test_update_while_an_iteration_is_in_flight(api):
    s1, s2 = EDITS["lambert_to_plastic"]()
    a = api.GPUVCM(s1, flavor="parity")
    a.run()
    a.iterate()
    a.update_scene(s2)  # drains the iteration in flight first
    _iterate(a, 3)
    b = _fresh(api, api.GPUVCM, s2, "parity")
    sa, sb = _vcm_state(a), _vcm_state(b)
    for key in sa:
        assert (rel_l2(sa[key], sb[key]) < 1e-6) if key == "film_light" else bit_equal(sa[key], sb[key]), key
    a.close()
    b.close()


@gpu
def test_update_is_bit_exact_against_the_oracle(api, oracle_mod):
    s1, s2 = _cornell(width=48, height=40), _cornell(_move_camera, width=48, height=40)
    a, _ = _updated(api, api.GPUVCM, s1, s2, "parity")
    o = oracle_mod.Oracle(s2)
    o.set_options(S.default_vcm_options())
    o.begin(0)
    o.run(3, threads=1)
    for bid, dt in VCM_BUFFERS + ((S.BUF_LIGHT_PATH_WAVELENGTH, np.float32), (S.BUF_CAMERA_GATHERED, np.float32)):
        assert bit_equal(a.buffer(bid, dt), o.buffer(bid, dt)), f"buffer {bid}"
    assert bit_equal(a.film(S.FILM_CAMERA)[..., :3], o.film(S.FILM_CAMERA)[..., :3])
    assert rel_l2(a.film(S.FILM_LIGHT)[..., :3], o.film(S.FILM_LIGHT)[..., :3]) < 1e-6
    a.close()


@gpu
def test_alternating_updates_do_not_grow_device_memory(api):
    import torch
    small, large = _plastic_box(lambert=True), _plastic_box(width=48, height=40)
    a = api.GPUPathTracing(small, flavor="fast")
    a.render(1)
    torch.cuda.synchronize()
    levels = []
    for cycle in range(10):
        for sd in (large, small):
            a.update_scene(sd)
            _iterate(a, 1)
        levels.append(torch.cuda.mem_get_info()[0])
    assert abs(levels[-1] - levels[0]) <= 16 << 20, [f"{(x - levels[0]) / 2**20:.1f} MB" for x in levels]
    a.close()


@gpu
def test_group_update_equals_a_fresh_group(api):
    s1, s2 = EDITS["lambert_to_plastic"]()
    f1, f2 = api.GPUVCMGroup(s2, lanes=2), api.GPUVCMGroup(s2, lanes=2)
    for f in (f1, f2):
        f.render(4)  # the lanes take iterations in any order: the combined film is a float sum in that order
    a = api.GPUVCMGroup(s1, lanes=2)
    a.render(2)
    info = a.update_scene(s2)
    assert info["kept"] & S.KEPT_GEOMETRY
    a.render(4)
    ra, r1, r2 = (g.film(S.FILM_RESULT)[..., :3] for g in (a, f1, f2))
    _within_fresh_spread(ra, r1, r2, "film_result")
    for g in (a, f1, f2):
        g.close()


# ---- the C++ adapters (host/gpu_vcm.hpp, host/gpu_pt.hpp) ------------------------------------------------------------------------------
NO_DEVICE_SRC = r'''
#include <cstdio>
#include "etx_tracer_b200/host/gpu_vcm.hpp"
#include "etx_tracer_b200/host/gpu_pt.hpp"
static_assert(sizeof(etxb_update_info) == 56, "etxb_update_info layout (structs.UPDATE_INFO)");
int main() {
  etxb_scene scene = {};
  etxb_camera camera = {};
  etxb::GPUVCM vcm(0);
  etxb::GPUPathTracing pt(0);
  if (vcm.enabled() || pt.enabled()) { std::puts("device present"); return 0; }
  etxb_update_info info = {};
  if (vcm.update_scene(&scene, sizeof(scene), &camera, sizeof(camera), 4, &info) == 0) return 1;
  if (pt.update_scene(&scene, sizeof(scene), &camera, sizeof(camera), 4, &info) == 0) return 2;
  if (vcm.can_run() || pt.can_run()) return 3;
  if (vcm.state() != etxb::GPUVCM::State::Stopped || pt.state() != etxb::GPUPathTracing::State::Stopped) return 4;
  if (etxb_update_scene(nullptr, &scene, sizeof(scene), &camera, sizeof(camera), &info) != ETXB_ERR_INVALID_ARGUMENT) return 5;
  if (etxb_group_update_scene(nullptr, &scene, sizeof(scene), &camera, sizeof(camera), &info) != ETXB_ERR_INVALID_ARGUMENT) return 6;
  std::puts("no-device contract ok");
  return 0;
}
'''


def _compile(tmp_path, name, code):
    lib = etx_build.lib_path("fast")
    if not os.path.exists(lib):
        etx_build.build(("fast",))
    src = tmp_path / f"{name}.cpp"
    src.write_text(code)
    exe = tmp_path / name
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-pthread", "-Wall", "-Werror", f"-I{ROOT}", str(src), lib, f"-Wl,-rpath,{os.path.dirname(lib)}", "-o", str(exe)])
    return str(exe)


def test_update_adapters_compile_and_fail_closed_without_device(tmp_path):
    exe = _compile(tmp_path, "u", NO_DEVICE_SRC)
    out = subprocess.run([exe], capture_output=True, text=True)
    assert out.returncode == 0, (out.returncode, out.stdout, out.stderr)


RENDER_SRC = r'''
// The application's camera drag on a real device: GPUVCM runs the scene, the camera is edited mid-run and update_scene restarts the render
// on the moved camera, which then renders to completion.
#include <chrono>
#include <cstdio>
#include <cstdint>
#include <thread>
#include <vector>
#include "etx_tracer_b200/host/gpu_vcm.hpp"
static std::vector<uint8_t> slurp(FILE* f, uint64_t n) { std::vector<uint8_t> v(n); if (n && fread(v.data(), 1, n, f) != n) v.clear(); return v; }
int main(int argc, char** argv) {
  FILE* f = fopen(argv[1], "rb");
  if (!f) return 1;
  uint64_t counts[10];
  if (fread(counts, 8, 10, f) != 10) return 2;
  etxb_scene scene; etxb_camera camera, moved;
  if (fread(&scene, sizeof(scene), 1, f) != 1 || fread(&camera, sizeof(camera), 1, f) != 1 || fread(&moved, sizeof(moved), 1, f) != 1) return 3;
  std::vector<std::vector<uint8_t>> arrays;
  for (int k = 0; k < 10; ++k) arrays.push_back(slurp(f, counts[k]));
  std::vector<uint8_t> xyz = slurp(f, 441 * 3 * 4), rgbr = slurp(f, 391 * 3 * 4), sobol = slurp(f, 256 * 256), scr = slurp(f, 128 * 128 * 8), rnk = slurp(f, 128 * 128 * 8);
  fclose(f);
  etxb_array_view* views[9] = {&scene.vertices, &scene.triangles, &scene.triangle_to_emitter, &scene.materials, &scene.emitter_profiles, &scene.emitter_instances,
                               &scene.images, &scene.mediums, &scene.spectrums};
  for (int k = 0; k < 9; ++k) views[k]->a = arrays[k].empty() ? nullptr : arrays[k].data();
  scene.emitters_distribution.values.a = arrays[9].data();
  etxb::GPUVCM vcm(0);
  if (!vcm.enabled()) return 4;
  if (vcm.upload_tables((const float*)xyz.data(), (const float*)rgbr.data(), sobol.data(), scr.data(), rnk.data()) != 0) return 5;
  if (vcm.commit_scene(&scene, sizeof(scene), &camera, sizeof(camera), 6) != 0) { std::printf("%s\n", vcm.status_str()); return 6; }
  vcm.run();
  bool moved_once = false;
  uint32_t pumps = 0;
  while (vcm.state() != etxb::GPUVCM::State::Stopped) {
    vcm.update();
    if (!moved_once && (vcm.status().completed_iterations >= 2)) {
      etxb_update_info info = {};
      if (vcm.update_scene(&scene, sizeof(scene), &moved, sizeof(moved), 6, &info) != 0) { std::printf("%s\n", vcm.status_str()); return 7; }
      if (vcm.state() != etxb::GPUVCM::State::Running) return 8;
      if (info.kept != (ETXB_KEPT_GEOMETRY | ETXB_KEPT_PATH_STATE)) return 9;
      moved_once = true;
    }
    std::this_thread::sleep_for(std::chrono::microseconds(200));
    if (++pumps > 2000000) return 10;
  }
  if (!moved_once || (vcm.status().completed_iterations != 6)) return 11;
  std::vector<float> film(size_t(moved.film_size[0]) * moved.film_size[1] * 4);
  if (vcm.read_film(ETXB_FILM_RESULT, film.data(), film.size() * 4) != 0) return 12;
  FILE* out = fopen(argv[2], "wb");
  fwrite(film.data(), 4, film.size(), out);
  fclose(out);
  return 0;
}
'''


@gpu
def test_cpp_adapter_follows_a_camera_move_mid_run(api, tmp_path):
    s1, s2 = _cornell(width=48, height=40, samples=6), _cornell(_move_camera, width=48, height=40, samples=6)
    sc = s1.scene
    names = ["vertices", "triangles", "triangle_to_emitter", "materials", "emitter_profiles", "emitter_instances", "images", "mediums", "spectrums"]
    sizes = [S.VERTEX.itemsize, S.TRIANGLE.itemsize, 4, S.MATERIAL.itemsize, S.EMITTER_PROFILE.itemsize, S.EMITTER.itemsize, S.IMAGE.itemsize, S.MEDIUM.itemsize,
             S.SPECTRUM.itemsize]
    blobs = []
    for n, sz in zip(names, sizes):
        cnt = int(sc[n]["count"][0])
        blobs.append(bytes((C.c_char * (cnt * sz)).from_address(int(sc[n]["a"][0]))) if cnt else b"")
    ne = int(sc["emitter_instances"]["count"][0])
    blobs.append(bytes((C.c_char * ((ne + 1) * S.DIST_ENTRY.itemsize)).from_address(int(sc["emitters_distribution"]["values"]["a"][0]))))
    ct, bn = scenes.tables("color_tables"), scenes.tables("bluenoise")
    with open(tmp_path / "scene.bin", "wb") as f:
        f.write(np.array([len(b) for b in blobs], dtype=np.uint64).tobytes())
        f.write(sc.tobytes())
        f.write(s1.camera.tobytes())
        f.write(s2.camera.tobytes())
        for b in blobs:
            f.write(b)
        f.write(np.ascontiguousarray(ct["xyz_441x3"], dtype=np.float32).tobytes())
        f.write(np.ascontiguousarray(ct["rgb_response_391x3"], dtype=np.float32).tobytes())
        for k in ("sobol", "scrambling_8", "ranking_8"):  # next_power(min(samples = 6, 256))
            f.write(np.ascontiguousarray(bn[k], dtype=np.uint8).tobytes())
    exe = _compile(tmp_path, "r", RENDER_SRC)
    out = subprocess.run([exe, str(tmp_path / "scene.bin"), str(tmp_path / "film.bin")], capture_output=True, text=True)
    assert out.returncode == 0, (out.returncode, out.stdout[-500:], out.stderr[-500:])
    film = np.fromfile(tmp_path / "film.bin", dtype=np.float32).reshape(s2.height, s2.width, 4)
    g = api.GPUVCM(s2, flavor="fast")
    g.render(6)
    ref = g.film(S.FILM_RESULT)
    g.close()
    assert rel_l2(film[..., :3], ref[..., :3]) < 1e-5  # the light image is a float-atomic sum
