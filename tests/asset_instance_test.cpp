// Compiles the C++ host mirror's instance entry points (GaussianSplatRenderer::CreateInstanceOf,
// GaussianSplatRendererGroup::AddInstance) against the C ABI and drives them.  Exit codes:
// 0 = every frame matched, 3 = no CUDA device (expected on a machine without one: the library must fail loudly), 1 = anything else.
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <vector>

#include "../unitygaussiansplatting_b200/host/GaussianSplatRenderer.hpp"

int main() {
  using namespace GaussianSplatting;
  const uint32_t n = 256;
  // one VeryHigh (all float32, no chunks) asset: splats on a ring in front of the camera
  std::vector<float> pos(n * 3), other(n * 4), color(2048 * 16 * 4, 0.0f), sh(n * 48, 0.0f);
  for (uint32_t i = 0; i < n; ++i) {
    float a = 6.2831853f * i / n;
    pos[i * 3] = 0.8f * std::cos(a); pos[i * 3 + 1] = 0.8f * std::sin(a); pos[i * 3 + 2] = 0.1f * std::sin(3.0f * a);
    uint32_t q = 511u | (511u << 10) | (511u << 20) | (3u << 30);   // ~identity rotation, 10.10.10.2
    std::memcpy(&other[i * 4], &q, 4);
    other[i * 4 + 1] = other[i * 4 + 2] = other[i * 4 + 3] = 0.05f;
    uint32_t t = (i & 0xFF) | ((i & 0xFE) << 7); t &= 0x5555; t = (t ^ (t >> 1)) & 0x3333; t = (t ^ (t >> 2)) & 0x0f0f;
    uint32_t tx = t & 0xF, ty = t >> 8;
    float *c = &color[(ty * 2048 + tx) * 4];
    c[0] = 1.0f; c[1] = 0.5f * (i & 1); c[2] = 0.25f; c[3] = 0.6f;
  }
  GsAssetDesc d{};
  d.splat_count = n;
  d.pos = pos.data(); d.pos_bytes = pos.size() * 4;
  d.other = other.data(); d.other_bytes = other.size() * 4;
  d.color = color.data(); d.color_bytes = color.size() * 4;
  d.sh = sh.data(); d.sh_bytes = sh.size() * 4;
  // twin owns the context and is destroyed last (locals go in reverse order); source and instance draw on its context
  GaussianSplatRenderer twin, source, instance;
  if (!twin.OnEnable(d)) return twin.context() == nullptr ? 3 : 1;
  if (!source.OnEnable(d, twin.context()) || !instance.CreateInstanceOf(source)) return 1;
  if (gs_asset_device_ptr(instance.asset(), 3) != gs_asset_device_ptr(source.asset(), 3) ||
      gs_asset_device_ptr(instance.asset(), 0) == gs_asset_device_ptr(source.asset(), 0)) {
    std::fprintf(stderr, "the instance does not share exactly the source's blobs\n");
    return 1;
  }
  CameraState cam{};
  const float f = 1.0f / std::tan(0.5f * 0.8f), zn = 0.3f, zf = 100.0f;
  float view[16] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, -1, 0, 0, 0, -3, 1};                 // camera at (0,0,-3) looking +z; row 2 negated
  float proj[16] = {f, 0, 0, 0, 0, -f, 0, 0, 0, 0, zn / (zf - zn), -1, 0, 0, zf * zn / (zf - zn), 0};   // reversed-z, y flipped
  std::memcpy(cam.worldToCameraMatrix.m, view, 64);
  std::memcpy(cam.gpuProjectionMatrix.m, proj, 64);
  cam.pixelWidth = 128; cam.pixelHeight = 128; cam.position[2] = -3.0f;
  auto draw = [&](GaussianSplatRenderer &r, std::vector<uint16_t> &rt) {
    rt.assign(128 * 128 * 4, 0);
    GsImage im{rt.data(), 128, 128, 0, GS_PIX_RGBA16F, GS_MEM_HOST};
    return r.SortAndRenderSplats(cam, &im);
  };
  auto lit = [](const std::vector<uint16_t> &rt) {
    size_t k = 0;
    for (size_t i = 3; i < rt.size(); i += 4) k += rt[i] != 0;
    return k;
  };
  // the instance is drawn with its own transform; the source draws in between, then is disabled, and the instance draws on
  std::vector<uint16_t> a, b, c;
  instance.localToWorldMatrix.m[12] = twin.localToWorldMatrix.m[12] = 0.3f;
  instance.worldToLocalMatrix.m[12] = twin.worldToLocalMatrix.m[12] = -0.3f;
  for (int pass = 0; pass < 2; ++pass) {
    if (!draw(twin, a) || !draw(instance, b)) return 1;
    if (lit(a) <= 100 || a != b) { std::fprintf(stderr, "instance frame %d differs from a separate upload's\n", pass); return 1; }
    if (pass == 0) {
      if (!draw(source, c) || c == a) return 1;
      source.OnDisable();
    }
  }
  std::printf("asset instance: frames equal a separate upload\n");
  // the group: member assets' instances (AddInstance) against AddObject's uploads, two contexts emulated on this device
  GaussianSplatRendererGroup grp;
  if (!grp.OnEnable(d, std::vector<int>{0, 0}, GS_GROUP_EMULATE)) return 1;
  GaussianSplatGroupObject *inst = grp.AddInstance(grp), *up = grp.AddObject(d);
  if (!inst || !up || gs_asset_device_ptr(inst->m_Assets[1], 4) != gs_asset_device_ptr(grp.asset(1), 4)) return 1;
  std::vector<uint16_t> g[4];
  for (auto &v : g) v.assign(128 * 128 * 4, 0);
  GsImage i0{g[0].data(), 128, 128, 0, GS_PIX_RGBA16F, GS_MEM_HOST}, i1{g[1].data(), 128, 128, 0, GS_PIX_RGBA16F, GS_MEM_HOST},
      i2{g[2].data(), 128, 128, 0, GS_PIX_RGBA16F, GS_MEM_HOST}, i3{g[3].data(), 128, 128, 0, GS_PIX_RGBA16F, GS_MEM_HOST};
  GsImage *r01[2] = {&i0, &i1}, *r23[2] = {&i2, &i3};
  inst->localToWorldMatrix.m[12] = up->localToWorldMatrix.m[12] = 0.3f;
  inst->worldToLocalMatrix.m[12] = up->worldToLocalMatrix.m[12] = -0.3f;
  if (!grp.SortAndRenderSplatsMulti(cam, {inst}, r01) || !grp.SortAndRenderSplatsMulti(cam, {up}, r23) || !grp.Sync()) return 1;
  if (lit(g[0]) <= 100 || g[0] != g[2] || g[1] != g[3] || g[0] != g[1]) { std::fprintf(stderr, "group instance frame differs\n"); return 1; }
  std::printf("asset instance: group instance equals an upload\n");
  return 0;
}
