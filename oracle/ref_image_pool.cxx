// The reference's OWN ImagePool (sources/etx/render/host/image_pool.cxx, compiled in place into libreference_loader.so by build_oracle.sh)
// behind one C export, for tests/test_reference_image.py: the float4 pixels the pool holds after add_from_file(file, 0, {}, {1, 1}), which is what
// the application's viewer shows as its reference image (raytracer/app.cxx:243-250).  TEST INFRASTRUCTURE, built by build_ref_image_pool.sh.
#include <etx/render/host/image_pool.hxx>
#include <etx/render/host/tasks.hxx>

#include <cstdint>
#include <cstring>

extern "C" {

// 0 and the pixels (rows as the pool stores them, Image::pixel read-out: RGBA8 as UNORM) when rgba holds w * h float4; 1 with w, h alone
int refpool_read(const char* file_name, uint32_t* width, uint32_t* height, float* rgba, uint64_t capacity) {
  etx::TaskScheduler scheduler;
  etx::ImagePool pool(scheduler);
  pool.init(4u);
  const uint32_t handle = pool.add_from_file(file_name, 0u, {}, {1.0f, 1.0f});
  const etx::Image& img = pool.get(handle);
  *width = img.isize.x, *height = img.isize.y;
  const uint64_t n = uint64_t(img.isize.x) * img.isize.y;
  int rc = 1;
  if ((rgba != nullptr) && (capacity >= n * 16u)) {
    for (uint64_t i = 0; i < n; ++i) {
      const auto p = img.pixel(uint32_t(i));
      memcpy(rgba + 4u * i, &p, 16u);
    }
    rc = 0;
  }
  pool.cleanup();
  return rc;
}

}  // extern "C"
