// film_io.cpp — what the application does with a finished film layer (SURVEY 8(f) N4): RTApplication::on_save_image_selected
// (sources/raytracer/app.cxx:261-295) writes either the float4 layer as an OpenEXR file (tinyexr SaveEXR, 4 float channels) or the
// tone-mapped layer as an 8-bit PNG (stb_image_write).  Neither third-party writer is used here: an EXR scan-line file without compression
// and a PNG with stored (uncompressed) deflate blocks are a few dozen lines each and every reader accepts them — tests/test_film_io.py reads
// them back with the reference's own tinyexr / stb_image (compiled into oracle/_ref/libreference_loader.so) and with zlib.
// Host-only code: no CUDA here; the tone-mapping itself runs on the device (k_film_tonemap, kernels_view.cuh) or through etxb_tonemap_rgba8.
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <vector>

#include "../../include/etx_b200.h"

namespace {

struct Bytes {
  std::vector<uint8_t> v;
  void raw(const void* p, size_t n) {
    const uint8_t* b = static_cast<const uint8_t*>(p);
    v.insert(v.end(), b, b + n);
  }
  void u8(uint8_t x) { v.push_back(x); }
  void le32(uint32_t x) {
    for (int k = 0; k < 4; ++k) v.push_back(uint8_t(x >> (8 * k)));
  }
  void le64(uint64_t x) {
    for (int k = 0; k < 8; ++k) v.push_back(uint8_t(x >> (8 * k)));
  }
  void be32(uint32_t x) {
    for (int k = 3; k >= 0; --k) v.push_back(uint8_t(x >> (8 * k)));
  }
  void str(const char* s) { raw(s, strlen(s) + 1); }
};

void exr_attribute(Bytes& b, const char* name, const char* type, const Bytes& value) {
  b.str(name);
  b.str(type);
  b.le32(uint32_t(value.v.size()));
  b.raw(value.v.data(), value.v.size());
}

bool write_file(const char* file_name, const Bytes& b) {
  FILE* f = fopen(file_name, "wb");
  if (!f) return false;
  const bool ok = fwrite(b.v.data(), 1, b.v.size(), f) == b.v.size();
  return (fclose(f) == 0) && ok;
}

uint32_t crc_table[256];
bool crc_ready = false;
uint32_t crc32(const uint8_t* p, size_t n, uint32_t crc = 0xffffffffu) {
  if (!crc_ready) {
    for (uint32_t i = 0; i < 256; ++i) {
      uint32_t c = i;
      for (int k = 0; k < 8; ++k) c = (c & 1u) ? (0xedb88320u ^ (c >> 1)) : (c >> 1);
      crc_table[i] = c;
    }
    crc_ready = true;
  }
  for (size_t i = 0; i < n; ++i) crc = crc_table[(crc ^ p[i]) & 0xffu] ^ (crc >> 8);
  return crc;
}

void png_chunk(Bytes& out, const char* type, const Bytes& data) {
  out.be32(uint32_t(data.v.size()));
  Bytes body;
  body.raw(type, 4);
  body.raw(data.v.data(), data.v.size());
  out.raw(body.v.data(), body.v.size());
  out.be32(crc32(body.v.data(), body.v.size()) ^ 0xffffffffu);
}

float linear_to_gamma(float value) {  // math.hxx:1040-1042
  return value <= 0.0031308f ? 12.92f * value : 1.055f * powf(value, 1.0f / 2.4f) - 0.055f;
}
float saturate(float v) { return (v > 0.0f) ? (v > 1.0f ? 1.0f : v) : 0.0f; }  // a NaN maps to 0

}  // namespace

extern "C" {

// SaveEXR(data, width, height, 4 components, fp16 = false, ...) as app.cxx:289 calls it: channels A, B, G, R as 32-bit floats, one scan line per
// block, no compression, increasing-y line order.  rgba = row-major float4, the film's own storage order (y already flipped, film.cxx:165,189).
int etxb_write_exr(const char* file_name, const float* rgba, uint32_t width, uint32_t height) {
  if (!file_name || !rgba || (width == 0u) || (height == 0u)) return ETXB_ERR_INVALID_ARGUMENT;
  Bytes b;
  b.le32(20000630u);  // magic
  b.le32(2u);         // version 2, single-part scan-line image
  {
    Bytes ch;
    for (const char* name : {"A", "B", "G", "R"}) {  // a chlist is sorted by channel name
      ch.str(name);
      ch.le32(2u);  // FLOAT
      ch.u8(0);     // pLinear
      ch.u8(0), ch.u8(0), ch.u8(0);
      ch.le32(1u), ch.le32(1u);  // x / y sampling
    }
    ch.u8(0);
    exr_attribute(b, "channels", "chlist", ch);
  }
  {
    Bytes c;
    c.u8(0);  // NO_COMPRESSION
    exr_attribute(b, "compression", "compression", c);
  }
  Bytes window;
  window.le32(0u), window.le32(0u), window.le32(width - 1u), window.le32(height - 1u);
  exr_attribute(b, "dataWindow", "box2i", window);
  exr_attribute(b, "displayWindow", "box2i", window);
  {
    Bytes lo;
    lo.u8(0);  // INCREASING_Y
    exr_attribute(b, "lineOrder", "lineOrder", lo);
  }
  const float one = 1.0f, zero = 0.0f;
  {
    Bytes f;
    f.raw(&one, 4);
    exr_attribute(b, "pixelAspectRatio", "float", f);
  }
  {
    Bytes f;
    f.raw(&zero, 4), f.raw(&zero, 4);
    exr_attribute(b, "screenWindowCenter", "v2f", f);
  }
  {
    Bytes f;
    f.raw(&one, 4);
    exr_attribute(b, "screenWindowWidth", "float", f);
  }
  b.u8(0);  // end of header
  const uint64_t line_bytes = uint64_t(width) * 16u, block_bytes = 8u + line_bytes;
  const uint64_t data_start = b.v.size() + uint64_t(height) * 8u;
  for (uint32_t y = 0; y < height; ++y) b.le64(data_start + uint64_t(y) * block_bytes);
  std::vector<float> plane(size_t(width) * 4u);
  static const int order[4] = {3, 2, 1, 0};  // A, B, G, R from RGBA
  for (uint32_t y = 0; y < height; ++y) {
    b.le32(y);
    b.le32(uint32_t(line_bytes));
    const float* row = rgba + size_t(y) * width * 4u;
    for (int c = 0; c < 4; ++c)
      for (uint32_t x = 0; x < width; ++x) plane[size_t(c) * width + x] = row[size_t(x) * 4u + order[c]];
    b.raw(plane.data(), plane.size() * 4u);  // x86 / the GPU box are little endian like the file format
  }
  return write_file(file_name, b) ? ETXB_OK : ETXB_ERR_INVALID_ARGUMENT;
}

// stbi_write_png(file, w, h, 4, data, 0) as app.cxx:283 calls it: 8-bit RGBA, no interlace; the zlib stream uses stored blocks
int etxb_write_png(const char* file_name, const uint8_t* rgba8, uint32_t width, uint32_t height) {
  if (!file_name || !rgba8 || (width == 0u) || (height == 0u)) return ETXB_ERR_INVALID_ARGUMENT;
  Bytes raw;  // filter byte 0 + the row
  raw.v.reserve((size_t(width) * 4u + 1u) * height);
  for (uint32_t y = 0; y < height; ++y) {
    raw.u8(0);
    raw.raw(rgba8 + size_t(y) * width * 4u, size_t(width) * 4u);
  }
  Bytes z;
  z.u8(0x78), z.u8(0x01);
  uint32_t a = 1u, s = 0u;  // adler32
  for (size_t i = 0; i < raw.v.size(); ++i) {
    a = (a + raw.v[i]) % 65521u;
    s = (s + a) % 65521u;
  }
  for (size_t at = 0; at < raw.v.size();) {
    const size_t n = std::min<size_t>(65535u, raw.v.size() - at);
    z.u8((at + n == raw.v.size()) ? 1 : 0);
    z.u8(uint8_t(n & 0xffu)), z.u8(uint8_t(n >> 8));
    z.u8(uint8_t(~n & 0xffu)), z.u8(uint8_t((~n >> 8) & 0xffu));
    z.raw(raw.v.data() + at, n);
    at += n;
  }
  z.be32((s << 16) | a);
  Bytes out;
  static const uint8_t signature[8] = {0x89, 'P', 'N', 'G', 0x0d, 0x0a, 0x1a, 0x0a};
  out.raw(signature, 8);
  Bytes ihdr;
  ihdr.be32(width), ihdr.be32(height);
  ihdr.u8(8), ihdr.u8(6), ihdr.u8(0), ihdr.u8(0), ihdr.u8(0);  // 8 bits, RGBA, deflate, adaptive filtering, no interlace
  png_chunk(out, "IHDR", ihdr);
  png_chunk(out, "IDAT", z);
  png_chunk(out, "IEND", Bytes{});
  return write_file(file_name, out) ? ETXB_OK : ETXB_ERR_INVALID_ARGUMENT;
}

// The tone map of the reference's LDR export (app.cxx:268-282; the viewer's shader does the same, render.cxx:307-320):
// 1 - exp(-exposure * c), sRGB transfer curve, 8 bits with truncation, alpha 255.  Host version (the device one is etxb_read_film_ldr).
int etxb_tonemap_rgba8(const float* rgba, uint64_t pixel_count, float exposure, uint8_t* out_rgba8) {
  if (!rgba || !out_rgba8) return ETXB_ERR_INVALID_ARGUMENT;
  for (uint64_t i = 0; i < pixel_count; ++i) {
    for (int c = 0; c < 3; ++c) {
      float tm = 1.0f - expf(-exposure * rgba[i * 4u + c]);
      out_rgba8[i * 4u + c] = static_cast<uint8_t>(255.0f * saturate(linear_to_gamma(tm)));
    }
    out_rgba8[i * 4u + 3u] = 255u;
  }
  return ETXB_OK;
}

}  // extern "C"
