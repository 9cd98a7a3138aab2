// asset_creator.cpp -- host-side packer + synthetic scene generator (libgsplat_asset.so).
//
// Produces the five byte blobs of a GaussianSplatAsset in exactly the layout the
// reference's importer writes (package/Editor/GaussianSplatAssetCreator.cs, cited per
// function below as E/...:line).  This is new code: a flat, OpenMP-parallel C++ pipeline
// over one contiguous record array, not a translation of the Burst job structs.
//
// The format's rules and encoders are gs_asset_format.h, shared with the GPU packer (gs_pack.cu).
// oracle/refcs/ compiles the reference's own C# and tests/test_reference_cs.py compares this file's bytes with it.
#include "../../include/gsplat_asset.h"
#include "gs_asset_format.h"

#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <limits>
#include <zlib.h>

#include <cstdio>
#include <string>
#include <vector>
#ifdef _OPENMP
#include <omp.h>
#include <parallel/algorithm>
#endif

int gsa_usable_threads();  // asset_cluster_bc7.cpp: OpenMP default capped by affinity mask and cgroup CPU quota

namespace {

using namespace gs;

// ---- counter-based RNG for the synthetic scenes (pcg hash, same family as the k-means') ----
struct Rng {
  uint32_t base;
  uint32_t ctr;
  Rng(uint32_t seed, uint32_t index) : base(pcg_hash(seed ^ pcg_hash(index * 0x9E3779B9u + 0x7F4A7C15u))), ctr(0) {}
  uint32_t next() { return pcg_hash(base + (ctr++) * 0x85EBCA6Bu); }
  float uniform() { return f32_from_bits(0x3f800000u | (next() >> 9)) - 1.0f; }  // [0,1)
  float range(float lo, float hi) { return lo + (hi - lo) * uniform(); }
  float normal() {  // Box-Muller
    float u1 = std::max(uniform(), 1.0e-7f);
    float u2 = uniform();
    return std::sqrt(-2.0f * std::log(u1)) * std::cos(6.2831853f * u2);
  }
};

inline float sigmoid(float v) { return 1.0f / (1.0f + std::exp(-v)); }  // R/GaussianUtils.cs:9-12

// R/GaussianUtils.cs:46-76
inline void pack_smallest3(const float qin[4], float out[4]) {
  float q[4] = {qin[0], qin[1], qin[2], qin[3]};
  float ax = std::fabs(q[0]), ay = std::fabs(q[1]), az = std::fabs(q[2]), aw = std::fabs(q[3]);
  int index = 0;
  float maxV = ax;
  if (ay > maxV) { index = 1; maxV = ay; }
  if (az > maxV) { index = 2; maxV = az; }
  if (aw > maxV) { index = 3; maxV = aw; }
  float r[4] = {q[0], q[1], q[2], q[3]};
  if (index == 0) { r[0] = q[1]; r[1] = q[2]; r[2] = q[3]; r[3] = q[0]; }  // yzwx
  if (index == 1) { r[0] = q[0]; r[1] = q[2]; r[2] = q[3]; r[3] = q[1]; }  // xzwy
  if (index == 2) { r[0] = q[0]; r[1] = q[1]; r[2] = q[3]; r[3] = q[2]; }  // xywz
  float sgn = (r[3] >= 0.0f) ? 1.0f : -1.0f;
  const float kSqrt2 = 1.41421356237f;
  for (int k = 0; k < 3; ++k) out[k] = ((r[k] * sgn) * kSqrt2) * 0.5f + 0.5f;
  out[3] = (float)index / 3.0f;
}

static_assert(sizeof(GsaInputSplat) == kRecFloats * 4, "InputSplatData must be 248 bytes");
static_assert(offsetof(GsaInputSplat, dc0) == kOffDc0 * 4 && offsetof(GsaInputSplat, sh) == kOffSh * 4 &&
                  offsetof(GsaInputSplat, opacity) == kOffOpacity * 4 && offsetof(GsaInputSplat, scale) == kOffScale * 4 &&
                  offsetof(GsaInputSplat, rot) == kOffRot * 4,
              "GsaInputSplat is the record emit_splat reads");

void normalize4(float q[4]) {
  float l = std::sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
  if (l < 1e-20f) { q[0] = q[1] = q[2] = 0; q[3] = 1; return; }
  for (int k = 0; k < 4; ++k) q[k] /= l;
}

}  // namespace

extern "C" {

uint64_t gsa_morton_encode3(uint32_t x, uint32_t y, uint32_t z) { return morton_encode3(x, y, z); }
uint32_t gsa_splat_index_to_texture_index(uint32_t idx) { return splat_index_to_texel(idx); }
void gsa_pack_smallest3(const float q[4], float out[4]) { pack_smallest3(q, out); }
uint32_t gsa_f32tof16(float v) { return unity_f32tof16(v); }

int gsa_generate(uint32_t kind, uint32_t n, uint32_t seed, GsaInputSplat *out) {
  if (!out || kind > GSA_SCENE_UNIFORM) return -1;
#pragma omp parallel for schedule(static) num_threads(gsa_usable_threads())
  for (int64_t ii = 0; ii < (int64_t)n; ++ii) {
    uint32_t i = (uint32_t)ii;
    Rng r(seed, i);
    GsaInputSplat s;
    std::memset(&s, 0, sizeof(s));
    float q[4] = {0, 0, 0, 1};
    if (kind == GSA_SCENE_LATTICE) {
      uint32_t k = i % 1000u;
      float lx = -1.0f + 2.0f * (float)(k % 10u) / 9.0f;
      float ly = -1.0f + 2.0f * (float)((k / 10u) % 10u) / 9.0f;
      float lz = -1.0f + 2.0f * (float)((k / 100u) % 10u) / 9.0f;
      float jx = r.range(-0.02f, 0.02f), jy = r.range(-0.02f, 0.02f), jz = r.range(-0.02f, 0.02f);
      s.pos[0] = lx + jx;
      s.pos[1] = ly + jy;
      s.pos[2] = (i & 1u) ? lz : lz + jz;  // odd splats keep the exact lattice z: deliberate depth ties
      for (int k2 = 0; k2 < 3; ++k2) s.scale[k2] = std::exp(r.range(std::log(0.01f), std::log(0.05f)));
      s.opacity = r.range(0.1f, 1.0f);
      for (int k2 = 0; k2 < 3; ++k2) s.dc0[k2] = r.uniform();
    } else if (kind == GSA_SCENE_CLUSTERED) {
      bool in_cluster = r.uniform() < 0.7f;
      if (in_cluster) {
        uint32_t cid = r.next() & 4095u;
        Rng c(seed ^ 0xC1057E25u, cid);
        float cx = c.range(-8.0f, 8.0f), cy = c.range(-2.0f, 3.0f), cz = c.range(-8.0f, 8.0f);
        float sig = c.range(0.05f, 0.6f);
        s.pos[0] = cx + sig * r.normal();
        s.pos[1] = cy + sig * r.normal();
        s.pos[2] = cz + sig * r.normal();
      } else {
        float d[3] = {r.normal(), r.normal(), r.normal()};
        float l = std::sqrt(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]) + 1e-12f;
        float rad = r.range(8.0f, 30.0f);
        for (int k2 = 0; k2 < 3; ++k2) s.pos[k2] = d[k2] / l * rad;
      }
      for (int k2 = 0; k2 < 3; ++k2) {
        float sc = std::exp(std::log(0.02f) + 0.7f * r.normal());
        s.scale[k2] = std::min(std::max(sc, 1.0e-3f), 2.0f);
      }
      for (int k2 = 0; k2 < 4; ++k2) q[k2] = r.normal();
      normalize4(q);
      s.opacity = sigmoid(2.5f * r.normal());
      for (int k2 = 0; k2 < 3; ++k2) s.dc0[k2] = r.uniform();
      for (int k2 = 0; k2 < 45; ++k2) s.sh[k2] = 0.05f * r.normal();
    } else {
      for (int k2 = 0; k2 < 3; ++k2) s.pos[k2] = r.range(-20.0f, 20.0f);
      for (int k2 = 0; k2 < 3; ++k2) s.scale[k2] = std::exp(r.range(std::log(0.005f), std::log(0.05f)));
      for (int k2 = 0; k2 < 4; ++k2) q[k2] = r.normal();
      normalize4(q);
      s.opacity = r.range(0.05f, 0.9f);
      for (int k2 = 0; k2 < 3; ++k2) s.dc0[k2] = r.uniform();
      for (int k2 = 0; k2 < 45; ++k2) s.sh[k2] = 0.05f * r.normal();
    }
    pack_smallest3(q, s.rot);
    out[i] = s;
  }
  return 0;
}

int gsa_calc_sizes(uint32_t n, uint32_t pf, uint32_t sf, uint32_t cf, uint32_t shf, GsaSizes *out) {
  return out && calc_sizes(n, pf, sf, cf, shf, out) ? 0 : -1;
}

int gsa_create_asset(GsaInputSplat *splats, uint32_t n, uint32_t pf, uint32_t sf, uint32_t cf, uint32_t shf,
                     void *pos_out, void *other_out, void *color_out, void *sh_out, void *chunks_out,
                     float *bounds_out) {
  GsaSizes sz;
  if (!splats || !pos_out || !other_out || !color_out || !sh_out) return -1;
  if (gsa_calc_sizes(n, pf, sf, cf, shf, &sz) != 0) return -4;
  const bool chunked = uses_chunks(pf, sf, cf, shf);
  if (chunked && !chunks_out) return -1;

  // ---- bounds (E/...:361-385) ----
  float bmin[3] = {INFINITY, INFINITY, INFINITY}, bmax[3] = {-INFINITY, -INFINITY, -INFINITY};
  for (uint32_t i = 0; i < n; ++i)
    for (int k = 0; k < 3; ++k) {
      bmin[k] = unity_min(bmin[k], splats[i].pos[k]);
      bmax[k] = unity_max(bmax[k], splats[i].pos[k]);
    }
  if (bounds_out) { std::memcpy(bounds_out, bmin, 12); std::memcpy(bounds_out + 3, bmax, 12); }

  // ---- Morton reorder (E/...:387-429): sort by (code, index) ----
  {
    const float kScaler = (float)((1 << 21) - 1);
    float inv[3];
    for (int k = 0; k < 3; ++k) inv[k] = 1.0f / (bmax[k] - bmin[k]);
    std::vector<std::pair<uint64_t, int32_t>> order(n);
#pragma omp parallel for schedule(static) num_threads(gsa_usable_threads())
    for (int64_t i = 0; i < (int64_t)n; ++i) {
      uint32_t ip[3];
      for (int k = 0; k < 3; ++k) {
        float p = (splats[i].pos[k] - bmin[k]) * inv[k] * kScaler;
        ip[k] = (p >= 0.0f && p < 4294967296.0f) ? (uint32_t)p : 0u;  // C# (uint) of NaN/negative is unspecified; 0 here
      }
      order[i] = {morton_encode3(ip[0], ip[1], ip[2]), (int32_t)i};
    }
#ifdef _OPENMP
    __gnu_parallel::sort(order.begin(), order.end(), __gnu_parallel::default_parallel_tag(gsa_usable_threads()));
#else
    std::sort(order.begin(), order.end());
#endif
    std::vector<GsaInputSplat> copy(splats, splats + n);
#pragma omp parallel for schedule(static) num_threads(gsa_usable_threads())
    for (int64_t i = 0; i < (int64_t)n; ++i) splats[i] = copy[order[i].second];
  }

  // ---- SH palette (E/...:284-291, 476-518): k-means over the raw (not yet chunk-normalised) SH vectors ----
  std::vector<int32_t> sh_labels;
  if (shf > 3) {
    const uint32_t k = sh_count(shf, n);
    static const float kPasses[5] = {0.3f, 0.4f, 0.5f, 0.8f, 1.2f};  // Cluster64k..4k, E/...:487-495
    std::vector<float> sh_data((size_t)n * 45), means((size_t)k * 45);
#pragma omp parallel for schedule(static) num_threads(gsa_usable_threads())
    for (int64_t i = 0; i < (int64_t)n; ++i) std::memcpy(&sh_data[(size_t)i * 45], splats[i].sh, 180);  // GatherSHs :431-440
    sh_labels.resize(n);
    if (gsa_kmeans(45, sh_data.data(), n, 2048, kPasses[shf - 4], means.data(), k, sh_labels.data()) != 0) return -4;
    uint8_t *tab = (uint8_t *)sh_out;  // ConvertSHClustersJob :443-468: 15 x half3 + one padding half3 = 96 bytes
    std::memset(tab, 0, (size_t)k * 96);
    for (uint32_t j = 0; j < k; ++j) {
      uint16_t h[45];
      for (int c = 0; c < 45; ++c) h[c] = (uint16_t)unity_f32tof16(means[(size_t)j * 45 + c]);
      std::memcpy(tab + (size_t)j * 96, h, 90);
    }
  }

  // ---- chunk min/max + normalise (E/...:520-639) ----
  if (chunked) {
    ChunkInfo *chunks = (ChunkInfo *)chunks_out;
    const int64_t chunk_count = (n + kChunkSize - 1) / kChunkSize;
#pragma omp parallel for schedule(dynamic, 64) num_threads(gsa_usable_threads())
    for (int64_t c = 0; c < chunk_count; ++c) {
      float mn[13], mx[13];   // 0..2 position, 3..5 scale, 6..9 colour (dc0 rgb, opacity), 10..12 SH channel
      for (int q = 0; q < 13; ++q) { mn[q] = INFINITY; mx[q] = -INFINITY; }
      uint32_t b = (uint32_t)std::min<int64_t>(c * kChunkSize, n), e = (uint32_t)std::min<int64_t>((c + 1) * kChunkSize, n);
      for (uint32_t i = b; i < e; ++i) {
        GsaInputSplat &s = splats[i];
        for (int k = 0; k < 3; ++k) s.scale[k] = (float)std::pow((double)s.scale[k], (double)(1.0f / 8.0f));
        s.opacity = square_centered01(s.opacity);
        const float v[10] = {s.pos[0], s.pos[1], s.pos[2], s.scale[0], s.scale[1], s.scale[2], s.dc0[0], s.dc0[1], s.dc0[2], s.opacity};
        for (int q = 0; q < 10; ++q) { mn[q] = unity_min(mn[q], v[q]); mx[q] = unity_max(mx[q], v[q]); }
        for (int j = 0; j < 15; ++j)
          for (int k = 0; k < 3; ++k) {
            mn[10 + k] = unity_min(mn[10 + k], s.sh[j * 3 + k]); mx[10 + k] = unity_max(mx[10 + k], s.sh[j * 3 + k]);
          }
      }
      for (int q = 0; q < 13; ++q) mx[q] = unity_max(mx[q], mn[q] + 1.0e-5f);
      chunks[c] = encode_chunk(mn, mx);
      for (uint32_t i = b; i < e; ++i) {
        GsaInputSplat &s = splats[i];
        for (int k = 0; k < 3; ++k) {
          s.pos[k] = (s.pos[k] - mn[k]) / (mx[k] - mn[k]);
          s.scale[k] = (s.scale[k] - mn[3 + k]) / (mx[3 + k] - mn[3 + k]);
          s.dc0[k] = (s.dc0[k] - mn[6 + k]) / (mx[6 + k] - mn[6 + k]);
        }
        s.opacity = (s.opacity - mn[9]) / (mx[9] - mn[9]);
        for (int j = 0; j < 15; ++j)
          for (int k = 0; k < 3; ++k) s.sh[j * 3 + k] = (s.sh[j * 3 + k] - mn[10 + k]) / (mx[10 + k] - mn[10 + k]);
      }
    }
  }

  // ---- positions, other, colour, SH (E/...:705-1066) ----
  std::memset(pos_out, 0, sz.pos_bytes);
  std::memset(other_out, 0, sz.other_bytes);
  std::memset(color_out, 0, sz.color_bytes);
  if (shf <= 3) std::memset(sh_out, 0, sz.sh_bytes);
  // BC7 is encoded from the float image, 4x4 texels at a time (E/...:887-912)
  std::vector<float> image;
  if (cf == 3) image.assign((size_t)sz.tex_width * sz.tex_height * 4, 0.0f);
  const EmitTarget to{(uint8_t *)pos_out, (uint8_t *)other_out, (uint8_t *)color_out, (uint8_t *)sh_out, image.data(), pf, sf, cf, shf};
#pragma omp parallel for schedule(static) num_threads(gsa_usable_threads())
  for (int64_t i = 0; i < (int64_t)n; ++i)
    emit_splat(to, (uint32_t)i, reinterpret_cast<const float *>(&splats[i]), shf > 3 ? (uint32_t)sh_labels[i] : 0u);
  if (cf == 3) {
    const uint32_t bw = sz.tex_width / 4, bh = sz.tex_height / 4;
#pragma omp parallel for schedule(static) num_threads(gsa_usable_threads())
    for (int64_t b = 0; b < (int64_t)bw * bh; ++b) {
      const uint32_t bx = (uint32_t)(b % bw), by = (uint32_t)(b / bw);
      float blk[64];
      for (int y = 0; y < 4; ++y)
        std::memcpy(&blk[y * 16], &image[((size_t)(by * 4 + y) * sz.tex_width + bx * 4) * 4], 64);
      gsa_bc7_encode_block(blk, (uint8_t *)color_out + (size_t)b * 16);
    }
  }
  return 0;
}


// ---- INRIA .ply reader (E/Utils/PLYFileReader.cs, E/Utils/GaussianFileReader.cs) --------------------------------
namespace {
struct PlyHeader {
  int64_t count = -1;
  uint32_t stride = 0;
  bool binary_le = false;
  std::vector<std::pair<std::string, int>> attrs;  // name, size in bytes (4 float, 8 double, 1 uchar, 0 unknown)
  std::vector<bool> is_float;
  long data_offset = 0;
  bool unsupported = false;
};

bool read_line(FILE *f, std::string &line) {
  line.clear();
  int c;
  bool any = false;
  while ((c = fgetc(f)) != EOF) {
    any = true;
    if (c == '\n') break;
    line.push_back((char)c);
  }
  if (!line.empty() && line.back() == '\r') line.pop_back();  // CRLF
  return any;
}

bool parse_ply_header(FILE *f, PlyHeader &h) {
  std::string line;
  for (int i = 0; i < 9000; ++i) {  // kMaxHeaderLines
    if (!read_line(f, line) || line == "end_header" || line.empty()) break;
    char a[64], b[64], c[64];
    if (sscanf(line.c_str(), "%63s %63s %63s", a, b, c) != 3) continue;
    const std::string t0 = a, t1 = b, t2 = c;
    if (t0 == "format" && t1 == "binary_little_endian" && t2 == "1.0") h.binary_le = true;
    if (t0 == "element" && t1 == "vertex") h.count = atoll(c);
    if (t0 == "property") {
      const int size = t1 == "float" ? 4 : t1 == "double" ? 8 : t1 == "uchar" ? 1 : 0;
      if (size == 0) h.unsupported = true;   // int / short / list ...: the importer's TypeToSize throws (E/Utils/PLYFileReader.cs:95-105)
      h.stride += size;
      h.attrs.push_back({t2, size});
      h.is_float.push_back(t1 == "float");
    }
  }
  h.data_offset = ftell(f);
  if (!h.binary_le || h.count < 0 || h.unsupported) return false;
  // the vertex block the header promises must exist in the file (an untrusted count must not size an allocation)
  const long here = h.data_offset;
  if (fseek(f, 0, SEEK_END) != 0) return false;
  const long end = ftell(f);
  fseek(f, here, SEEK_SET);
  if (end < here || (uint64_t)(end - here) < (uint64_t)h.count * (uint64_t)h.stride) return false;
  return true;
}

const char *kSplatAttrs[62] = {
    "x", "y", "z", "nx", "ny", "nz", "f_dc_0", "f_dc_1", "f_dc_2",
    "f_rest_0", "f_rest_1", "f_rest_2", "f_rest_3", "f_rest_4", "f_rest_5", "f_rest_6", "f_rest_7", "f_rest_8", "f_rest_9",
    "f_rest_10", "f_rest_11", "f_rest_12", "f_rest_13", "f_rest_14", "f_rest_15", "f_rest_16", "f_rest_17", "f_rest_18", "f_rest_19",
    "f_rest_20", "f_rest_21", "f_rest_22", "f_rest_23", "f_rest_24", "f_rest_25", "f_rest_26", "f_rest_27", "f_rest_28", "f_rest_29",
    "f_rest_30", "f_rest_31", "f_rest_32", "f_rest_33", "f_rest_34", "f_rest_35", "f_rest_36", "f_rest_37", "f_rest_38", "f_rest_39",
    "f_rest_40", "f_rest_41", "f_rest_42", "f_rest_43", "f_rest_44",
    "opacity", "scale_0", "scale_1", "scale_2", "rot_0", "rot_1", "rot_2", "rot_3"};
const char *kRequired[14] = {"x", "y", "z", "f_dc_0", "f_dc_1", "f_dc_2", "opacity", "scale_0", "scale_1", "scale_2",
                             "rot_0", "rot_1", "rot_2", "rot_3"};
}  // namespace

int64_t gsa_ply_vertex_count(const char *path) {
  FILE *f = path ? fopen(path, "rb") : nullptr;
  if (!f) return -1;
  PlyHeader h;
  const bool ok = parse_ply_header(f, h);
  fclose(f);
  if (!ok) return -2;
  for (const char *req : kRequired) {  // CheckPLYAttributes, GaussianFileReader.cs:73-80
    bool found = false;
    for (size_t i = 0; i < h.attrs.size(); ++i) found |= h.attrs[i].first == req && h.is_float[i];
    if (!found) return -3;
  }
  return h.count;
}

// ExportPlyFile, E/GaussianSplatRendererEditor.cs:394-445: header with the 62 float properties in kSplatAttrs order (LF line
// ends), then every record that is neither deleted (bit set in `deleted_bits`, may be NULL) nor marked cut (nor != 0 --
// CSExportData's "skipped for export" flag).  `records` are raw .ply attribute values, i.e. gs_export_splats' output.
int64_t gsa_ply_write(const char *path, const float *records, uint32_t n, const uint32_t *deleted_bits) {
  if (!path || (!records && n)) return -1;
  auto alive = [&](uint32_t i) {
    const bool deleted = deleted_bits && (deleted_bits[i >> 5] & (1u << (i & 31)));
    const float *r = records + (size_t)i * 62;
    const bool cut = (r[3] * r[3] + r[4] * r[4] + r[5] * r[5]) > 0.0f;
    return !deleted && !cut;
  };
  int64_t count = 0;
  for (uint32_t i = 0; i < n; ++i) count += alive(i) ? 1 : 0;
  FILE *f = fopen(path, "wb");
  if (!f) return -1;
  std::string header = "ply\nformat binary_little_endian 1.0\nelement vertex " + std::to_string(count) + "\n";
  for (const char *name : kSplatAttrs) header += std::string("property float ") + name + "\n";
  header += "end_header\n";
  bool ok = fwrite(header.data(), 1, header.size(), f) == header.size();
  for (uint32_t i = 0; i < n && ok; ++i)
    if (alive(i)) ok = fwrite(records + (size_t)i * 62, 4, 62, f) == 62;
  ok = (fclose(f) == 0) && ok;
  return ok ? count : -1;
}

static int ply_read_impl(const char *path, GsaInputSplat *out, uint32_t capacity);
int gsa_ply_read(const char *path, GsaInputSplat *out, uint32_t capacity) {
  try {
    return ply_read_impl(path, out, capacity);
  } catch (...) {   // nothing may cross the C boundary (std::bad_alloc on a huge file)
    return -5;
  }
}
static int ply_read_impl(const char *path, GsaInputSplat *out, uint32_t capacity) {
  const int64_t n = gsa_ply_vertex_count(path);
  if (n < 0) return (int)n;
  if (!out || (uint64_t)n > capacity) return -1;
  FILE *f = fopen(path, "rb");
  if (!f) return -1;
  PlyHeader h;
  parse_ply_header(f, h);
  std::vector<int> src_off(62, -1);  // PLYDataToSplats, GaussianFileReader.cs:82-169
  {
    int off = 0;
    for (size_t i = 0; i < h.attrs.size(); ++i) {
      if (h.is_float[i])
        for (int k = 0; k < 62; ++k)
          if (h.attrs[i].first == kSplatAttrs[k] && src_off[k] < 0) src_off[k] = off;
      off += h.attrs[i].second;
    }
  }
  std::vector<uint8_t> raw((size_t)n * h.stride);
  fseek(f, h.data_offset, SEEK_SET);
  const size_t got = fread(raw.data(), 1, raw.size(), f);
  fclose(f);
  if (got != raw.size()) return -4;
#pragma omp parallel for schedule(static) num_threads(gsa_usable_threads())
  for (int64_t i = 0; i < n; ++i) {
    float d[62];
    const uint8_t *src = raw.data() + (size_t)i * h.stride;
    for (int k = 0; k < 62; ++k) {
      d[k] = 0.0f;
      if (src_off[k] >= 0) std::memcpy(&d[k], src + src_off[k], 4);
    }
    // ReorderSHs: f_rest is channel-major (15 R, 15 G, 15 B) -> 15 x RGB  (:183-205)
    float tmp[45];
    for (int j = 0; j < 15; ++j) { tmp[j * 3] = d[9 + j]; tmp[j * 3 + 1] = d[9 + j + 15]; tmp[j * 3 + 2] = d[9 + j + 30]; }
    std::memcpy(&d[9], tmp, sizeof(tmp));
    GsaInputSplat s;
    std::memcpy(&s, d, sizeof(s));
    // LinearizeData (:207-232): rot_0..3 = (w,x,y,z) -> normalise -> (x,y,z,w) -> smallest-three
    float q[4] = {s.rot[0], s.rot[1], s.rot[2], s.rot[3]};
    // math.normalize(wxyz).yzwx: rsqrt(dot(q, q)) * q, a multiply by the reciprocal length, not a divide
    const float rlen = 1.0f / std::sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
    const float qn[4] = {rlen * q[1], rlen * q[2], rlen * q[3], rlen * q[0]};
    pack_smallest3(qn, s.rot);
    for (int k = 0; k < 3; ++k) s.scale[k] = std::fabs(std::exp(s.scale[k]));      // LinearScale
    for (int k = 0; k < 3; ++k) s.dc0[k] = s.dc0[k] * 0.2820948f + 0.5f;           // SH0ToColor
    s.opacity = 1.0f / (1.0f + std::exp(-s.opacity));                               // Sigmoid
    out[i] = s;
  }
  return 0;
}


// ---- Niantic .spz reader (E/Utils/SPZFileReader.cs) -----------------------------------------------------------
namespace {
struct SpzHeader { uint32_t magic, version, numPoints, sh_fracbits_flags_reserved; };
int spz_open(const char *path, gzFile *gz, SpzHeader *h) {
  *gz = path ? gzopen(path, "rb") : nullptr;
  if (!*gz) return -1;
  if (gzread(*gz, h, 16) != 16 || h->magic != 0x5053474eu || h->version != 2u) { gzclose(*gz); return -2; }   // :38-47
  return 0;
}
}  // namespace

int64_t gsa_spz_vertex_count(const char *path) {
  gzFile gz;
  SpzHeader h;
  const int rc = spz_open(path, &gz, &h);
  if (rc) return rc;
  gzclose(gz);
  return (int64_t)h.numPoints;
}

int gsa_spz_read(const char *path, GsaInputSplat *out, uint32_t capacity) {
  gzFile gz;
  SpzHeader h;
  int rc = spz_open(path, &gz, &h);
  if (rc) return rc;
  const int64_t n = h.numPoints;
  const int shLevel = (int)(h.sh_fracbits_flags_reserved & 0xFF), fractBits = (int)((h.sh_fracbits_flags_reserved >> 8) & 0xFF);
  if (n < 1 || n > 10000000 || shLevel < 0 || shLevel > 3 || fractBits < 0 || fractBits > 24 || !out || (uint64_t)n > capacity) {  // :70-75
    gzclose(gz);
    return -3;
  }
  const int shCoeffs = shLevel == 1 ? 3 : shLevel == 2 ? 8 : shLevel == 3 ? 15 : 0;  // :54-64
  std::vector<uint8_t> pos((size_t)n * 9), alpha((size_t)n), col((size_t)n * 3), scale((size_t)n * 3), rot((size_t)n * 3),
      sh((size_t)n * 3 * shCoeffs);
  auto rd = [&](std::vector<uint8_t> &v) {   // gzread takes an unsigned int length: read in slices
    size_t done = 0;
    while (done < v.size()) {
      const unsigned want = (unsigned)std::min<size_t>(v.size() - done, 1u << 30);
      const int got = gzread(gz, v.data() + done, want);
      if (got <= 0) return false;
      done += (size_t)got;
    }
    return true;
  };
  const bool ok = rd(pos) && rd(alpha) && rd(col) && rd(scale) && rd(rot) && rd(sh);  // stream order, :87-93
  gzclose(gz);
  if (!ok) return -4;
  const float fractScale = 1.0f / (float)(1 << fractBits);
#pragma omp parallel for schedule(static) num_threads(gsa_usable_threads())
  for (int64_t i = 0; i < n; ++i) {  // UnpackDataJob, :125-195
    GsaInputSplat s;
    std::memset(&s, 0, sizeof(s));
    for (int k = 0; k < 3; ++k) {
      const size_t b = ((size_t)i * 3 + k) * 3;
      int32_t fx = pos[b] | (pos[b + 1] << 8) | (pos[b + 2] << 16);
      if (fx & 0x800000) fx |= (int32_t)0xff000000;   // 24-bit sign extension
      s.pos[k] = (float)fx * fractScale;
      s.scale[k] = std::fabs(std::exp((float)scale[(size_t)i * 3 + k] / 16.0f - 10.0f));
    }
    const float x = (float)rot[(size_t)i * 3] * (1.0f / 127.5f) - 1.0f, y = (float)rot[(size_t)i * 3 + 1] * (1.0f / 127.5f) - 1.0f,
                z = (float)rot[(size_t)i * 3 + 2] * (1.0f / 127.5f) - 1.0f;
    const float w = std::sqrt(std::max(0.0f, 1.0f - (x * x + y * y + z * z)));
    const float len = std::sqrt(x * x + y * y + z * z + w * w);
    const float q[4] = {x / len, y / len, z / len, w / len};
    pack_smallest3(q, s.rot);
    s.opacity = (float)alpha[(size_t)i] / 255.0f;
    for (int k = 0; k < 3; ++k) {
      float c = (float)col[(size_t)i * 3 + k] / 255.0f - 0.5f;
      c /= 0.15f;
      s.dc0[k] = c * 0.2820948f + 0.5f;   // SH0ToColor
    }
    const size_t shIdx = (size_t)i * shCoeffs * 3;
    for (int j = 0; j < shCoeffs * 3; ++j) s.sh[j] = ((float)sh[shIdx + j] - 128.0f) / 128.0f;
    out[i] = s;
  }
  return 0;
}

}  // extern "C"
