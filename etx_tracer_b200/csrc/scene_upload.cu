// scene_upload.cu — etxb_upload_scene and etxb_update_scene (Raytracing::commit_changes, sources/etx/rt/rt.cxx:58-88): the checks of a scene,
// the content hashes of its bulk arrays, and their device copies.  Host code only: the last step of a commit, the film and path-state buffers
// the kernels size, is module.cu's (commit_path_state).  The stages are declared in context.cuh; etxb_group_update_scene (group.cu) runs them
// once for all its lanes.
#include <cstring>

#include "bvh_build_device.h"
#include "context.cuh"

namespace {

// 128-bit content hash of a byte range, chained through `seed`: four independent 64-bit multiply-rotate lanes over 32-byte stripes (the
// round of xxHash64), a zero-padded tail, and two differently mixed 64-bit digests of the lanes and the length.  It detects edits, not
// adversaries.
constexpr uint64_t kHashP1 = 0x9E3779B185EBCA87ull, kHashP2 = 0xC2B2AE3D27D4EB4Full, kHashP3 = 0x165667B19E3779F9ull, kHashP4 = 0x85EBCA77C2B2AE63ull;
inline uint64_t rotl64(uint64_t x, int r) { return (x << r) | (x >> (64 - r)); }
inline uint64_t hash_round(uint64_t acc, uint64_t w) { return rotl64(acc + w * kHashP2, 31) * kHashP1; }
inline uint64_t hash_mix(uint64_t h) {
  h ^= h >> 33;
  h *= kHashP2;
  h ^= h >> 29;
  h *= kHashP3;
  return h ^ (h >> 32);
}
Hash128 hash128(const void* data, size_t bytes, Hash128 seed) {
  const uint8_t* p = static_cast<const uint8_t*>(data);
  uint64_t v[4] = {seed.lo + kHashP1 + kHashP2, seed.hi + kHashP2, seed.lo ^ kHashP3, seed.hi - kHashP1};
  size_t i = 0;
  for (; i + 32 <= bytes; i += 32) {
    uint64_t w[4];
    memcpy(w, p + i, 32);
    for (int k = 0; k < 4; ++k) v[k] = hash_round(v[k], w[k]);
  }
  uint64_t tail[4] = {0, 0, 0, 0};
  if (bytes > i) memcpy(tail, p + i, bytes - i);
  for (int k = 0; k < 4; ++k) v[k] = hash_round(v[k], tail[k]);
  const uint64_t a = rotl64(v[0], 1) + rotl64(v[1], 7) + rotl64(v[2], 12) + rotl64(v[3], 18);
  const uint64_t b = (v[0] * kHashP4) ^ rotl64(v[1], 29) ^ (v[2] * kHashP3) ^ rotl64(v[3], 43);
  return {hash_mix(a ^ (uint64_t(bytes) * kHashP4)), hash_mix(b + uint64_t(bytes) * kHashP1)};
}

bool material_class_supported_host(uint32_t cls) { return cls <= ETXB_MAT_VOID; }

// A Distribution over `size` items holds size + 1 entries (DistributionBuilder allocates the closing {0, 0, 1} entry, distribution_builder.hxx:8-14,
// 52) while `values.count` says `size` (the reference's loader) or size + 1 (hosts that count the closing entry): both are accepted, and the
// device always gets the size + 1 entries.
bool distribution_covers(uint64_t count, uint64_t size) { return (count == size) || (count == size + 1u); }

bool image_has_table(const etxb_image& im) {
  return (im.y_distribution.values.a != nullptr) && distribution_covers(im.y_distribution.values.count, im.isize[1]) && (im.x_distributions.count == im.isize[1]);
}
size_t image_pixel_bytes(const etxb_image& im) { return size_t(im.isize[0]) * im.isize[1] * (im.format == 1u ? 16 : 4); }

// Every check of the upload but the BVH depth (prepare_bvh), and the scene-class flags.  What the device path does not cover yet fails
// loudly (no CPU fallback); every index the host builder and the kernels follow is checked: a malformed scene is an error, not an
// out-of-bounds read.
int validate_scene(etxb_ctx* ctx, const etxb_scene& s, const etxb_camera& cam, SceneClass& c) {
  if (cam.cls > 1u) return fail(ctx, ETXB_ERR_INVALID_ARGUMENT, "unknown camera class %u", cam.cls);
  if (cam.lens_image != ETXB_INVALID_INDEX) {
    if (cam.lens_image >= s.images.count) return fail(ctx, ETXB_ERR_INVALID_ARGUMENT, "camera lens image index out of range");
    const auto& lens = static_cast<const etxb_image*>(s.images.a)[cam.lens_image];
    if (!distribution_covers(lens.y_distribution.values.count, lens.isize[1])) return fail(ctx, ETXB_ERR_INVALID_ARGUMENT, "camera lens image has no sampling table");
  }
  const auto* mats = static_cast<const etxb_material*>(s.materials.a);
  for (uint64_t i = 0; i < s.materials.count; ++i) {
    const etxb_material& m = mats[i];
    if (!material_class_supported_host(m.cls)) return fail(ctx, ETXB_ERR_UNSUPPORTED, "material %llu: class %u is not supported on the device yet", (unsigned long long)i, m.cls);
    if (m.diffuse_variation > 2u) return fail(ctx, ETXB_ERR_INVALID_ARGUMENT, "material %llu: unknown diffuse_variation %u", (unsigned long long)i, m.diffuse_variation);
    if (m.subsurface.cls > 2u) return fail(ctx, ETXB_ERR_INVALID_ARGUMENT, "material %llu: unknown subsurface class %u", (unsigned long long)i, m.subsurface.cls);
    if (m.subsurface.cls != 0) {
      if (s.subsurface_exit_material >= s.materials.count) return fail(ctx, ETXB_ERR_INVALID_ARGUMENT, "material %llu uses subsurface scattering but scene.subsurface_exit_material is not set", (unsigned long long)i);
      if ((m.subsurface.image_index != ETXB_INVALID_INDEX) && (m.subsurface.image_index >= s.images.count))
        return fail(ctx, ETXB_ERR_INVALID_ARGUMENT, "material %llu: subsurface image index out of range", (unsigned long long)i);
    }
    uint32_t imgs[] = {m.reflectance.image_index, m.scattering.image_index, m.emission.image_index, m.roughness.image_index, m.normal_image_index, m.thinfilm.thickness_image};
    for (uint32_t im : imgs)
      if ((im != ETXB_INVALID_INDEX) && (im >= s.images.count)) return fail(ctx, ETXB_ERR_INVALID_ARGUMENT, "material %llu: image index %u out of range", (unsigned long long)i, im);
    if (((m.int_medium != ETXB_INVALID_INDEX) && (m.int_medium >= s.mediums.count)) || ((m.ext_medium != ETXB_INVALID_INDEX) && (m.ext_medium >= s.mediums.count)))
      return fail(ctx, ETXB_ERR_INVALID_ARGUMENT, "material %llu: medium index out of range", (unsigned long long)i);
  }
  c = {};
  for (uint64_t i = 0; i < s.materials.count; ++i) {
    const etxb_material& m = mats[i];
    bool lambert = (m.cls == ETXB_MAT_DIFFUSE) && (m.diffuse_variation == 0);
    bool smooth = (std::max(m.roughness.value[0], m.roughness.value[1]) <= 1.0e-4f) && (m.roughness.image_index == ETXB_INVALID_INDEX);
    bool always_delta = (((m.cls == ETXB_MAT_DIELECTRIC) || (m.cls == ETXB_MAT_CONDUCTOR)) && smooth) || (m.cls == ETXB_MAT_THINFILM) || (m.cls == ETXB_MAT_MIRROR) ||
                        (m.cls == ETXB_MAT_VOID);
    if (!lambert && !always_delta) c.stochastic = true;
  }
  const auto* emitters = static_cast<const etxb_emitter*>(s.emitter_instances.a);
  for (uint64_t i = 0; i < s.emitter_instances.count; ++i) {
    if (emitters[i].cls > 2u) return fail(ctx, ETXB_ERR_INVALID_ARGUMENT, "emitter %llu: unknown class %u", (unsigned long long)i, emitters[i].cls);
    if (emitters[i].cls == 1u) {
      const auto& prof = static_cast<const etxb_emitter_profile*>(s.emitter_profiles.a)[emitters[i].profile];
      if (prof.emission.image_index >= s.images.count) return fail(ctx, ETXB_ERR_INVALID_ARGUMENT, "environment emitter %llu has no image", (unsigned long long)i);
      const auto& img = static_cast<const etxb_image*>(s.images.a)[prof.emission.image_index];
      if (!distribution_covers(img.y_distribution.values.count, img.isize[1])) return fail(ctx, ETXB_ERR_INVALID_ARGUMENT, "environment emitter %llu: image has no sampling table", (unsigned long long)i);
    }
  }
  // media (medium.hxx:8-47)
  const auto* meds = static_cast<const etxb_medium*>(s.mediums.a);
  for (uint64_t i = 0; i < s.mediums.count; ++i) {
    const etxb_medium& md = meds[i];
    if (md.cls == 1u) {
      size_t n = size_t(md.dimensions[0]) * md.dimensions[1] * md.dimensions[2];
      if ((n == 0) || (md.density.count != n)) return fail(ctx, ETXB_ERR_INVALID_ARGUMENT, "medium %llu: density grid does not match its dimensions", (unsigned long long)i);
    } else if (md.cls != 0u) {
      return fail(ctx, ETXB_ERR_INVALID_ARGUMENT, "medium %llu: unknown class %u", (unsigned long long)i, md.cls);
    }
  }
  for (uint64_t i = 0; i < s.materials.count; ++i) {
    if (mats[i].cls == ETXB_MAT_BOUNDARY) c.boundaries = true;
    if (mats[i].subsurface.cls != 0) c.subsurface = true;
  }
  if ((cam.medium_index != ETXB_INVALID_INDEX) && (cam.medium_index >= s.mediums.count)) return fail(ctx, ETXB_ERR_INVALID_ARGUMENT, "camera medium index out of range");
  // deferred shadow rays (ShadowBatch, dvcm.cuh) need: no alpha test that can reject, no Boundary surfaces / media (transmittance is 0 or 1),
  // no BSDF whose evaluation draws from the sampler, no subsurface exits
  c.plain = !c.boundaries && !c.subsurface && (s.mediums.count == 0) && (cam.medium_index == ETXB_INVALID_INDEX);
  bool no_alpha = true;
  const auto* all_images = static_cast<const etxb_image*>(s.images.a);
  for (uint64_t i = 0; no_alpha && (i < s.materials.count); ++i) {
    if (mats[i].opacity != 1.0f) no_alpha = false;
    uint32_t im = mats[i].scattering.image_index;
    if ((im != ETXB_INVALID_INDEX) && (all_images[im].options & kImageHasAlpha)) no_alpha = false;
  }
  c.opaque = c.plain && no_alpha;
  c.deferred = c.opaque && !c.stochastic;
  // images: pixels + flattened row/column CDFs (image.hxx:8-50)
  for (uint64_t i = 0; i < s.images.count; ++i) {
    const etxb_image& im = all_images[i];
    if ((im.format != 1u) && (im.format != 2u)) return fail(ctx, ETXB_ERR_INVALID_ARGUMENT, "image %llu: unknown pixel format %u", (unsigned long long)i, im.format);
    if (size_t(im.isize[0]) * im.isize[1] == 0) return fail(ctx, ETXB_ERR_INVALID_ARGUMENT, "image %llu is empty", (unsigned long long)i);
    if (image_has_table(im)) {
      const auto* rows = static_cast<const etxb_distribution*>(im.x_distributions.a);
      for (uint32_t y = 0; y < im.isize[1]; ++y)
        if (!distribution_covers(rows[y].values.count, im.isize[0])) return fail(ctx, ETXB_ERR_INVALID_ARGUMENT, "image %llu: row %u distribution has %llu entries", (unsigned long long)i, y, (unsigned long long)rows[y].values.count);
    }
  }
  if (s.emitter_instances.count == 0) return fail(ctx, ETXB_ERR_INVALID_ARGUMENT, "scene has no emitters");
  const auto* spectra = static_cast<const etxb_spectrum*>(s.spectrums.a);
  for (uint64_t i = 0; i < s.spectrums.count; ++i) {
    const etxb_spectrum& sp = spectra[i];
    if (sp.entry_count != 441) return fail(ctx, ETXB_ERR_UNSUPPORTED, "spectrum %llu has %u entries; the loader's 441-entry 390..830 nm grid is required", (unsigned long long)i, sp.entry_count);
    for (uint32_t k = 0; k < 441; ++k)
      if (sp.entries[k].wavelength != float(390 + k)) return fail(ctx, ETXB_ERR_UNSUPPORTED, "spectrum %llu is not on the integer 390..830 nm grid", (unsigned long long)i);
  }
  // geometry
  const auto* tris = static_cast<const etxb_triangle*>(s.triangles.a);
  for (uint64_t i = 0; i < s.triangles.count; ++i) {
    const etxb_triangle& t = tris[i];
    if ((t.i[0] >= s.vertices.count) || (t.i[1] >= s.vertices.count) || (t.i[2] >= s.vertices.count))
      return fail(ctx, ETXB_ERR_INVALID_ARGUMENT, "triangle %llu: vertex index out of range", (unsigned long long)i);
    if (t.material_index >= s.materials.count) return fail(ctx, ETXB_ERR_INVALID_ARGUMENT, "triangle %llu: material index %u out of range", (unsigned long long)i, t.material_index);
  }
  if (s.triangle_to_emitter.count != s.triangles.count)
    return fail(ctx, ETXB_ERR_INVALID_ARGUMENT, "triangle_to_emitter has %llu entries for %llu triangles", (unsigned long long)s.triangle_to_emitter.count, (unsigned long long)s.triangles.count);
  const auto* t2e = static_cast<const uint32_t*>(s.triangle_to_emitter.a);
  for (uint64_t i = 0; i < s.triangle_to_emitter.count; ++i)
    if ((t2e[i] != ETXB_INVALID_INDEX) && (t2e[i] >= s.emitter_instances.count)) return fail(ctx, ETXB_ERR_INVALID_ARGUMENT, "triangle %llu: emitter index out of range", (unsigned long long)i);
  for (uint64_t i = 0; i < s.emitter_instances.count; ++i) {
    if (emitters[i].profile >= s.emitter_profiles.count) return fail(ctx, ETXB_ERR_INVALID_ARGUMENT, "emitter %llu: profile index out of range", (unsigned long long)i);
    if ((emitters[i].cls == 0u) && (emitters[i].triangle_index >= s.triangles.count)) return fail(ctx, ETXB_ERR_INVALID_ARGUMENT, "area emitter %llu: triangle index out of range", (unsigned long long)i);
  }
  if (!distribution_covers(s.emitters_distribution.values.count, s.emitter_instances.count))
    return fail(ctx, ETXB_ERR_INVALID_ARGUMENT, "emitter distribution has %llu entries for %llu emitters", (unsigned long long)s.emitters_distribution.values.count, (unsigned long long)s.emitter_instances.count);
  if ((s.pixel_sampler_image != 0xffffffffu) && (s.pixel_sampler_image >= s.images.count)) return fail(ctx, ETXB_ERR_INVALID_ARGUMENT, "pixel sampler image out of range");
  if (size_t(cam.film_size[0]) * cam.film_size[1] == 0) return fail(ctx, ETXB_ERR_INVALID_ARGUMENT, "empty film");
  return ETXB_OK;
}

// a device-to-device copy into `dst`, sized as `src`
template <class T>
int copy_device(etxb_ctx* ctx, DevBuf<T>& dst, const DevBuf<T>& src) {
  CUDA_OK(ctx, dst.alloc(src.count));
  if (src.count) CUDA_OK(ctx, cudaMemcpyAsync(dst.ptr, src.ptr, src.bytes(), cudaMemcpyDeviceToDevice, ctx->stream));
  return ETXB_OK;
}

// An update keeps the device copy of image or density grid i when its content hash is the one last committed (`committed`: empty on an
// upload) and the copy has the size the new scene asks for
bool keep_by_hash(const std::vector<Hash128>& committed, const std::vector<Hash128>& now, uint64_t i, size_t held, size_t needed) {
  return (i < committed.size()) && (committed[i] == now[i]) && (held == needed);
}

// ---- commit_scene's steps, in the order it runs them; the film and path-state buffers are the last (commit_path_state, module.cu) ----------
// 1. media: dense density grids go to HBM as they are
int commit_media(etxb_ctx* ctx, const etxb_scene& s, const SceneHashes& old, const ScenePrep& p, etxb_update_info& st) {
  const auto* meds = static_cast<const etxb_medium*>(s.mediums.a);
  std::vector<DMedium> dmeds(s.mediums.count);
  ctx->medium_density.resize(s.mediums.count);
  for (uint64_t i = 0; i < s.mediums.count; ++i) {
    const etxb_medium& md = meds[i];
    DMedium& dm = dmeds[i];
    dm = {};
    dm.bounds_min = {md.bounds_min[0], md.bounds_min[1], md.bounds_min[2]};
    dm.bounds_max = {md.bounds_max[0], md.bounds_max[1], md.bounds_max[2]};
    dm.cls = md.cls;
    dm.enable_explicit_connections = md.enable_explicit_connections;
    dm.absorption_index = md.absorption_index;
    dm.scattering_index = md.scattering_index;
    dm.phase_function_g = md.phase_function_g;
    dm.max_sigma = md.max_sigma;
    dm.dim_x = md.dimensions[0];
    dm.dim_y = md.dimensions[1];
    dm.dim_z = md.dimensions[2];
    DevBuf<float>& grid = ctx->medium_density[i];
    if (md.cls == 1u) {
      size_t n = size_t(dm.dim_x) * dm.dim_y * dm.dim_z;
      if (keep_by_hash(old.grids, p.hashes.grids, i, grid.count, n)) {
        st.grids_kept += 1;
      } else {
        CUDA_OK(ctx, grid.alloc(n));
        CUDA_OK(ctx, cudaMemcpyAsync(grid.ptr, md.density.a, n * 4, cudaMemcpyHostToDevice, ctx->stream));
        st.grids_uploaded += 1;
      }
      dm.density = grid.ptr;
    } else {
      grid.release();
    }
  }
  if (int rc = upload(ctx, ctx->mediums, dmeds.data(), dmeds.size())) return rc;
  ctx->dscene.mediums = ctx->mediums.ptr;
  ctx->dscene.medium_count = uint32_t(dmeds.size());
  return ETXB_OK;
}

// 2. images: pixels + flattened row/column CDFs (image.hxx:8-50)
int commit_images(etxb_ctx* ctx, const etxb_scene& s, const SceneHashes& old, const ScenePrep& p, etxb_update_info& st) {
  const auto* imgs = static_cast<const etxb_image*>(s.images.a);
  std::vector<DImage> dimgs(s.images.count);
  ctx->image_pixels.resize(s.images.count);
  ctx->image_dists.resize(s.images.count * 2);
  for (uint64_t i = 0; i < s.images.count; ++i) {
    const etxb_image& im = imgs[i];
    DImage& di = dimgs[i];
    di = {};
    const size_t bytes = image_pixel_bytes(im);
    const bool table = image_has_table(im);
    DevBuf<uint8_t>& pixels = ctx->image_pixels[i];
    DevBuf<uint8_t>& x_dist = ctx->image_dists[i * 2];
    DevBuf<uint8_t>& y_dist = ctx->image_dists[i * 2 + 1];
    if (keep_by_hash(old.images, p.hashes.images, i, pixels.count, bytes)) {
      st.images_kept += 1;
    } else {
      CUDA_OK(ctx, pixels.alloc(bytes));
      CUDA_OK(ctx, cudaMemcpyAsync(pixels.ptr, im.pixels.a, bytes, cudaMemcpyHostToDevice, ctx->stream));
      x_dist.release();
      y_dist.release();
      if (table) {
        size_t nx = size_t(im.isize[0]) + 1u, ny = size_t(im.isize[1]) + 1u;
        std::vector<etxb_distribution_entry> flat(nx * im.isize[1]);
        const auto* rows = static_cast<const etxb_distribution*>(im.x_distributions.a);
        for (uint32_t y = 0; y < im.isize[1]; ++y) memcpy(flat.data() + size_t(y) * nx, rows[y].values.a, nx * sizeof(etxb_distribution_entry));
        CUDA_OK(ctx, x_dist.alloc(flat.size() * sizeof(etxb_distribution_entry)));
        CUDA_OK(ctx, cudaMemcpy(x_dist.ptr, flat.data(), flat.size() * sizeof(etxb_distribution_entry), cudaMemcpyHostToDevice));
        CUDA_OK(ctx, y_dist.alloc(ny * sizeof(etxb_distribution_entry)));
        CUDA_OK(ctx, cudaMemcpy(y_dist.ptr, im.y_distribution.values.a, ny * sizeof(etxb_distribution_entry), cudaMemcpyHostToDevice));
      }
      st.images_uploaded += 1;
    }
    di.pixels_f32 = (im.format == 1u) ? reinterpret_cast<const float4*>(pixels.ptr) : nullptr;
    di.pixels_u8 = (im.format == 2u) ? reinterpret_cast<const uchar4*>(pixels.ptr) : nullptr;
    di.fsize_x = im.fsize[0]; di.fsize_y = im.fsize[1];
    di.offset_x = im.offset[0]; di.offset_y = im.offset[1];
    di.scale_x = im.scale[0]; di.scale_y = im.scale[1];
    di.isize_x = im.isize[0]; di.isize_y = im.isize[1];
    di.normalization = im.normalization;
    di.options = im.options;
    di.format = im.format;
    if (table) {
      di.x_dist = reinterpret_cast<const etxb_distribution_entry*>(x_dist.ptr);
      di.y_dist = reinterpret_cast<const etxb_distribution_entry*>(y_dist.ptr);
      di.has_distribution = 1;
    }
  }
  if (int rc = upload(ctx, ctx->images, dimgs.data(), dimgs.size())) return rc;
  ctx->dscene.images = ctx->images.ptr;
  ctx->dscene.image_count = uint32_t(dimgs.size());
  return ETXB_OK;
}

// 3. the spectra and the small arrays, copied again on every call
int commit_tables(etxb_ctx* ctx, const etxb_scene& s) {
  const auto* spectra = static_cast<const etxb_spectrum*>(s.spectrums.a);
  std::vector<DSpectrum> dspec(s.spectrums.count);
  for (uint64_t i = 0; i < s.spectrums.count; ++i) {
    for (uint32_t k = 0; k < 441; ++k) dspec[i].power[k] = spectra[i].entries[k].power;
    memcpy(dspec[i].rgb, spectra[i].integrated, 12);
  }
  if (int rc = upload(ctx, ctx->tri_emitter, static_cast<const uint32_t*>(s.triangle_to_emitter.a), size_t(s.triangle_to_emitter.count))) return rc;
  if (int rc = upload(ctx, ctx->materials, static_cast<const etxb_material*>(s.materials.a), size_t(s.materials.count))) return rc;
  if (int rc = upload(ctx, ctx->profiles, static_cast<const etxb_emitter_profile*>(s.emitter_profiles.a), size_t(s.emitter_profiles.count))) return rc;
  if (int rc = upload(ctx, ctx->emitters, static_cast<const etxb_emitter*>(s.emitter_instances.a), size_t(s.emitter_instances.count))) return rc;
  if (int rc = upload(ctx, ctx->spectra, dspec.data(), dspec.size())) return rc;
  if (int rc = upload(ctx, ctx->emitter_dist, static_cast<const etxb_distribution_entry*>(s.emitters_distribution.values.a), size_t(s.emitter_instances.count) + 1u))
    return rc;
  DeviceScene& d = ctx->dscene;
  d.tri_emitter = ctx->tri_emitter.ptr;
  d.materials = ctx->materials.ptr;
  d.emitter_profiles = ctx->profiles.ptr;
  d.emitters = ctx->emitters.ptr;
  d.spectra = ctx->spectra.ptr;
  d.emitter_dist = ctx->emitter_dist.ptr;
  return ETXB_OK;
}

// 4. geometry: the vertices, triangles and BVH2 of a new geometry are copied from the prep, a kept one stays; then the 4-wide tree (product
// build, scenes with stochastic BSDFs).  `keep_wide`: the tree was kept with the geometry.
int commit_geometry(etxb_ctx* ctx, ScenePrep& p, bool keep_geometry, bool reuse, bool& keep_wide) {
  DeviceScene& d = ctx->dscene;
  if (!keep_geometry) {
    if (int rc = copy_device(ctx, ctx->vertices, p.vertices)) return rc;
    if (int rc = copy_device(ctx, ctx->triangles, p.triangles)) return rc;
    if (int rc = copy_device(ctx, ctx->bvh_nodes, p.bvh_nodes)) return rc;
    if (int rc = copy_device(ctx, ctx->bvh_tris, p.bvh_tris)) return rc;
    d.bvh_node_count = uint32_t(p.bvh_nodes.count);
  }
  d.vertices = ctx->vertices.ptr;
  d.triangles = ctx->triangles.ptr;
  d.bvh_nodes = ctx->bvh_nodes.ptr;
  d.bvh_tris = ctx->bvh_tris.ptr;
  keep_wide = false;
#if !(defined(ETXB_PARITY) && ETXB_PARITY)
  // a geometry whose 4-wide tree the traversal stack cannot hold keeps that verdict with it: an update that keeps the geometry does not
  // collapse the tree again only to reject it
  if (!keep_geometry) ctx->wide_rejected = false;
  keep_wide = keep_geometry && ctx->has_stochastic_merge && ((d.wide_nodes != nullptr) || ctx->wide_rejected);
#endif
  if (!keep_wide) {
    d.wide_nodes = nullptr;
    d.wide_node_count = 0;
    if (reuse) ctx->wide_nodes.release();
  }
#if !(defined(ETXB_PARITY) && ETXB_PARITY)
  if (ctx->has_stochastic_merge && !keep_wide) {
    // the sampler streams of such a scene's stochastic stages are the product build's own already: its traversal kernels may meet candidates in
    // another order, so they walk the 4-wide quantised form of the tree (dwide.cuh); Lambert / delta scenes keep the oracle's candidate order
    if (!p.have_wide) {
      // collapsed on the device from the committed BVH2 (new or kept: bvh_build_device.cu, the tree of build_wide_bvh)
      auto t0 = std::chrono::steady_clock::now();
      WideNode* wide = nullptr;
      uint32_t count = 0;
      CUDA_OK(ctx, build_wide_bvh_device(ctx->bvh_nodes.ptr, d.bvh_node_count, ctx->stream, &wide, &count, &p.max_stack));
      adopt(p.wide, wide, count);
      p.have_wide = true;
      const double seconds = seconds_since(t0);
      ctx->kernel_ms[K_BVH_WIDE] += float(seconds * 1.0e3);
      ctx->kernel_count[K_BVH_WIDE] += 1;
      p.bvh_seconds += seconds;
    }
    if (p.max_stack < uint32_t(kWideStackSize)) {
      if (int rc = copy_device(ctx, ctx->wide_nodes, p.wide)) return rc;
      d.wide_nodes = ctx->wide_nodes.ptr;
      d.wide_node_count = uint32_t(p.wide.count);
    } else {
      ctx->wide_rejected = true;
    }
  }
#endif
  return ETXB_OK;
}

// 5. the scene's constants and class into DeviceScene and the context
void commit_constants(etxb_ctx* ctx, const etxb_scene& s, const etxb_camera& cam, const SceneClass& c) {
  DeviceScene& d = ctx->dscene;
  d.has_boundaries = c.boundaries ? 1 : 0;
  d.has_subsurface = c.subsurface ? 1 : 0;
  d.subsurface_exit_material = s.subsurface_exit_material;
  d.deferred_shadow_rays = c.deferred ? 1u : 0u;
  d.emitter_count = uint32_t(s.emitter_instances.count);
  d.triangle_count = uint32_t(s.triangles.count);
  d.emitter_total_weight = s.emitters_distribution.total_weight;
  memcpy(d.env_emitters, s.environment_emitters, sizeof(d.env_emitters));
  d.env_emitter_count = s.environment_emitter_count;
  d.bounding_sphere_center = {s.bounding_sphere_center[0], s.bounding_sphere_center[1], s.bounding_sphere_center[2]};
  d.bounding_sphere_radius = s.bounding_sphere_radius;
  d.min_path_length = s.min_path_length;
  d.max_path_length = s.max_path_length;
  d.samples = s.samples;
  d.random_path_termination = s.random_path_termination;
  d.spectral = (s.flags & ETXB_SCENE_SPECTRAL) ? 1u : 0u;
  d.spectrum_count = uint32_t(s.spectrums.count);
  d.default_dielectric_eta = s.default_dielectric_eta;
  d.default_conductor_eta = s.default_conductor_eta;
  d.default_conductor_k = s.default_conductor_k;
  d.camera = cam;
  ctx->spectral = d.spectral != 0;
  ctx->pixel_sampler_image = s.pixel_sampler_image;
  ctx->pixel_sampler_radius = s.pixel_sampler_radius;
  ctx->noise_threshold = s.noise_threshold;
  ctx->radiance_clamp = s.radiance_clamp;
  ctx->scene_samples = s.samples;
}

// etxb_upload_scene (reuse = false: the scene that was there is dropped first, and every buffer is allocated and copied again) and
// etxb_update_scene (reuse = true: a scene already on the context keeps what the new one shares with it; refused with a communicator)
int load_scene(etxb_ctx* ctx, const void* scene_blob, uint64_t scene_bytes, const void* camera_blob, uint64_t camera_bytes, bool reuse, etxb_update_info* info) {
  const auto t0 = std::chrono::steady_clock::now();
  if (info) memset(info, 0, sizeof(*info));
  if (!ctx || !scene_blob || !camera_blob) return ETXB_ERR_INVALID_ARGUMENT;
  if (int rc = check_scene_args(ctx, scene_bytes, camera_bytes)) return rc;
  if (reuse && (ctx->comm != nullptr)) return fail(ctx, ETXB_ERR_UNSUPPORTED, "etxb_update_scene: a context with a communicator takes a new scene through etxb_upload_scene");
  ctx_drain(ctx);
  cudaSetDevice(ctx->device);
  if (!reuse) ctx->scene_ready = false;
  const etxb_scene& s = *static_cast<const etxb_scene*>(scene_blob);
  const etxb_camera& cam = *static_cast<const etxb_camera*>(camera_blob);
  ScenePrep p;
  if (int rc = prepare_scene(ctx, s, cam, p)) return rc;
  int rc = commit_scene(ctx, s, cam, p, reuse && ctx->scene_ready, info);
  if (info) info->total_seconds = seconds_since(t0);
  return rc;
}

}  // namespace

namespace etxb_internal __attribute__((visibility("hidden"))) {

int check_scene_args(etxb_ctx* ctx, uint64_t scene_bytes, uint64_t camera_bytes) {
  if (scene_bytes != sizeof(etxb_scene) || camera_bytes != sizeof(etxb_camera))
    return fail(ctx, ETXB_ERR_INVALID_ARGUMENT, "scene/camera size mismatch: got %llu/%llu, expected %zu/%zu", (unsigned long long)scene_bytes,
      (unsigned long long)camera_bytes, sizeof(etxb_scene), sizeof(etxb_camera));
  if (!ctx->xyz_table.ptr) return fail(ctx, ETXB_ERR_NOT_READY, "etxb_upload_color_tables must be called before etxb_upload_scene");
  return ETXB_OK;
}

// validate_scene + the content hashes of the arrays commit_scene may keep on the device: the vertices and triangles (one geometry
// hash), each image (pixels, sampling tables, scalar fields) and each density grid (values and dimensions)
int prepare_scene(etxb_ctx* ctx, const etxb_scene& s, const etxb_camera& cam, ScenePrep& p) {
  if (int rc = validate_scene(ctx, s, cam, p.cls)) return rc;
  auto t0 = std::chrono::steady_clock::now();
  SceneHashes& h = p.hashes;
  auto hash = [&p](const void* data, size_t bytes, Hash128 seed) {
    p.bytes_hashed += bytes;
    return hash128(data, bytes, seed);
  };
  h.geometry = hash(s.vertices.a, s.vertices.count * sizeof(etxb_vertex), {});
  h.geometry = hash(s.triangles.a, s.triangles.count * sizeof(etxb_triangle), h.geometry);
  h.images.assign(s.images.count, {});
  const auto* imgs = static_cast<const etxb_image*>(s.images.a);
  for (uint64_t i = 0; i < s.images.count; ++i) {
    const etxb_image& im = imgs[i];
    const bool table = image_has_table(im);
    const float fields[] = {im.fsize[0], im.fsize[1], im.offset[0], im.offset[1], im.scale[0], im.scale[1], im.normalization};
    const uint32_t ifields[] = {im.isize[0], im.isize[1], im.options, im.format, table ? 1u : 0u};
    Hash128 x = hash(fields, sizeof(fields), {});
    x = hash(ifields, sizeof(ifields), x);
    x = hash(im.pixels.a, image_pixel_bytes(im), x);
    if (table) {
      x = hash(im.y_distribution.values.a, (size_t(im.isize[1]) + 1u) * sizeof(etxb_distribution_entry), x);
      const auto* rows = static_cast<const etxb_distribution*>(im.x_distributions.a);
      for (uint32_t y = 0; y < im.isize[1]; ++y) x = hash(rows[y].values.a, (size_t(im.isize[0]) + 1u) * sizeof(etxb_distribution_entry), x);
    }
    h.images[i] = x;
  }
  h.grids.assign(s.mediums.count, {});
  const auto* meds = static_cast<const etxb_medium*>(s.mediums.a);
  for (uint64_t i = 0; i < s.mediums.count; ++i) {
    if (meds[i].cls != 1u) continue;
    h.grids[i] = hash(meds[i].dimensions, sizeof(meds[i].dimensions), {});
    h.grids[i] = hash(meds[i].density.a, meds[i].density.count * sizeof(float), h.grids[i]);
  }
  h.valid = true;
  p.fingerprint_seconds = seconds_since(t0);
  return ETXB_OK;
}

static_assert(sizeof(DTriangle) == sizeof(etxb_triangle), "triangle layout");

// A new geometry's vertices and triangles on the device, its BVH2 built there (bvh_build_device.cu: the tree of build_bvh), and the check of
// its depth against the traversal stack.  Everything goes into the prep's own buffers: a refusal or a CUDA error leaves the committed scene as it was.
int prepare_bvh(etxb_ctx* ctx, const etxb_scene& s, ScenePrep& p) {
  if (p.have_bvh) return ETXB_OK;
  auto t0 = std::chrono::steady_clock::now();
  const auto* verts = static_cast<const etxb_vertex*>(s.vertices.a);
  std::vector<DVertex> dverts(s.vertices.count);
  for (uint64_t i = 0; i < s.vertices.count; ++i) {
    const etxb_vertex& v = verts[i];
    dverts[i].pos_u = make_float4(v.pos[0], v.pos[1], v.pos[2], v.tex[0]);
    dverts[i].nrm_v = make_float4(v.nrm[0], v.nrm[1], v.nrm[2], v.tex[1]);
    dverts[i].tan = make_float4(v.tan[0], v.tan[1], v.tan[2], 0.0f);
    dverts[i].btn = make_float4(v.btn[0], v.btn[1], v.btn[2], 0.0f);
  }
  if (int rc = upload(ctx, p.vertices, dverts.data(), dverts.size())) return rc;
  if (int rc = upload(ctx, p.triangles, reinterpret_cast<const DTriangle*>(s.triangles.a), size_t(s.triangles.count))) return rc;
  const auto b0 = std::chrono::steady_clock::now();
  DeviceBvhOut out;
  CUDA_OK(ctx, build_bvh_device(reinterpret_cast<const float*>(p.vertices.ptr), sizeof(DVertex), reinterpret_cast<const uint32_t*>(p.triangles.ptr), sizeof(DTriangle),
    uint32_t(s.triangles.count), false, ctx->stream, out));
  adopt(p.bvh_nodes, out.nodes, out.node_count);
  adopt(p.bvh_tris, reinterpret_cast<float4*>(out.tri_pos), size_t(out.slot_count) * 3u);
  p.max_depth = out.max_depth;
  ctx->bvh_build_seconds = seconds_since(b0);
  ctx->kernel_ms[K_BVH_BUILD] += float(ctx->bvh_build_seconds * 1.0e3);
  ctx->kernel_count[K_BVH_BUILD] += 1;
  p.bvh_seconds += seconds_since(t0);
  p.have_bvh = true;
  if (p.max_depth >= uint32_t(kBvhStackSize)) return fail(ctx, ETXB_ERR_UNSUPPORTED, "BVH depth %u exceeds the traversal stack (%d)", p.max_depth, kBvhStackSize);
  return ETXB_OK;
}

bool geometry_kept(const etxb_ctx* ctx, const ScenePrep& p, bool reuse) { return reuse && ctx->hashes.valid && (ctx->hashes.geometry == p.hashes.geometry); }

// The device side of an upload (reuse = false: every buffer is allocated and copied again) or of an update (reuse = true: what the
// hashes show unchanged stays, path-state buffers of the same size stay).  Runs after prepare_scene, so only CUDA errors remain: they
// leave the scene not ready.  Ends with etxb_begin(ctx, 0).
int commit_scene(etxb_ctx* ctx, const etxb_scene& s, const etxb_camera& cam, ScenePrep& p, bool reuse, etxb_update_info* info) {
  const bool keep_geometry = geometry_kept(ctx, p, reuse);
  if (!keep_geometry)
    if (int rc = prepare_bvh(ctx, s, p)) return rc;
  SceneHashes old;  // what an update may keep
  if (reuse && ctx->hashes.valid) old = std::move(ctx->hashes);
  ctx->hashes = {};
  ctx->scene_ready = false;
  etxb_update_info st = {};
  ctx->has_stochastic_merge = p.cls.stochastic;
  ctx->plain_scene = p.cls.plain;
  ctx->opaque_scene = p.cls.opaque;
  bool keep_wide = false;
  uint32_t allocations = 0;
  if (int rc = commit_media(ctx, s, old, p, st)) return rc;
  if (int rc = commit_images(ctx, s, old, p, st)) return rc;
  if (int rc = commit_tables(ctx, s)) return rc;
  if (int rc = commit_geometry(ctx, p, keep_geometry, reuse, keep_wide)) return rc;
  commit_constants(ctx, s, cam, p.cls);
  if (int rc = commit_path_state(ctx, cam, reuse, &allocations)) return rc;
  CUDA_OK(ctx, cudaStreamSynchronize(ctx->stream));
  ctx->hashes = p.hashes;
  ctx->scene_ready = true;
  if (info) {
    st.kept = (keep_geometry ? ETXB_KEPT_GEOMETRY : 0u) | ((keep_wide && (ctx->dscene.wide_nodes != nullptr)) ? ETXB_KEPT_WIDE_TREE : 0u) |
              (allocations == 0 ? ETXB_KEPT_PATH_STATE : 0u);
    st.fingerprint_seconds = p.fingerprint_seconds;
    st.bytes_hashed = p.bytes_hashed;
    st.bvh_seconds = p.bvh_seconds;
    *info = st;
  }
  return etxb_begin(ctx, 0);
}

}  // namespace etxb_internal

int etxb_upload_scene(etxb_ctx* ctx, const void* scene_blob, uint64_t scene_bytes, const void* camera_blob, uint64_t camera_bytes) {
  return load_scene(ctx, scene_blob, scene_bytes, camera_blob, camera_bytes, false, nullptr);
}

int etxb_update_scene(etxb_ctx* ctx, const void* scene_blob, uint64_t scene_bytes, const void* camera_blob, uint64_t camera_bytes, etxb_update_info* info) {
  return load_scene(ctx, scene_blob, scene_bytes, camera_blob, camera_bytes, true, info);
}
