// ref_cs_harness.cpp -- C entry points around the reference importer's own packing code compiled for the CPU (see
// build_ref_cs.py, cs_shim.hpp).  TEST INFRASTRUCTURE ONLY.  The driver below is GaussianSplatAssetCreator.CreateAsset's
// sequence (E/GaussianSplatAssetCreator.cs:272-314) and the Create*Data methods around their jobs (:641-658, :812-861,
// :887-932, :1046-1066), restated without file I/O, the data hash, SH clustering and BC7 compression: bounds, Morton
// reorder, chunks when any format is lossy (isUsingChunks, :54-58), then positions, other, colour and SH.
#include "cs_shim.hpp"

namespace cs {
thread_local long g_conv_events = 0;
}

namespace refcs {
using namespace cs;
#include "ref_cs_gen.inc"
}  // namespace refcs

using namespace cs;
using namespace refcs;
typedef GaussianSplatAsset GSA;

static_assert(sizeof(InputSplatData) == 248, "InputSplatData layout");
static_assert(sizeof(GSA::ChunkInfo) == 64 && sizeof(GSA::SHTableItemFloat32) == 192 && sizeof(GSA::SHTableItemFloat16) == 96 &&
              sizeof(GSA::SHTableItemNorm11) == 60 && sizeof(GSA::SHTableItemNorm6) == 32, "the reference's blob layouts");

namespace {
bool clustered(int shf) { return shf >= (int)GSA::SHFormat::Cluster64k; }

// Runs job.Execute(i) for i < n and sets bit `bit` of flags[i] where a conversion in that call was out of range
template <class J> void run_marked(J &job, int n, uint8_t *flags, uint8_t bit) {
  for (int i = 0; i < n; ++i) {
    g_conv_events = 0;
    job.Execute(i);
    if (g_conv_events && flags) flags[i] |= bit;
  }
}
}  // namespace

extern "C" {

#define REF_API __attribute__((visibility("default")))

// Blob sizes as CreateAsset allocates them: chunk, pos, other (with the SH index a clustered format appends), colour
// (uncompressed formats; BC7 is one byte per texel), SH (clustered: the palette).  Texture width and height follow.
REF_API void ref_cs_sizes(int n, int pf, int sf, int cf, int shf, int64_t out[7]) {
  const bool chunks = pf != 0 || sf != 0 || cf != 0 || shf != 0;   // isUsingChunks
  out[0] = chunks ? GSA::CalcChunkDataSize(n) : 0;
  out[1] = GSA::CalcPosDataSize(n, (GSA::VectorFormat)pf);
  out[1] = GaussianSplatAssetCreator::NextMultipleOf((int)out[1], 8);
  const int ofs = GSA::GetOtherSizeNoSHIndex((GSA::VectorFormat)sf) + (clustered(shf) ? 2 : 0);
  out[2] = GaussianSplatAssetCreator::NextMultipleOf(n * ofs, 8);
  out[3] = GSA::CalcColorDataSize(n, (GSA::ColorFormat)cf);
  out[4] = GSA::CalcSHDataSize(n, (GSA::SHFormat)shf);
  const std::pair<int, int> wh = GSA::CalcTextureSize(n);
  out[5] = wh.first;
  out[6] = wh.second;
}

// CreateAsset on `splats` (consumed: reordered and chunk-normalised in place).  Writes every blob ref_cs_sizes sizes,
// except the BC7 colour image (cf 3) and, for clustered SH, the palette and the per-splat index (left zero in `other`).
// bounds: min xyz, max xyz.  conv_rec[i] (output order): bit 0 / 1 / 2 -- a float -> integer conversion of splat i's
// position / other / SH record was out of range; conv_rows[y]: the same for colour texture row y.  Returns the number of
// out-of-range conversions of the Morton codes (each makes the order itself a convention), or -1 on bad arguments.
REF_API long ref_cs_create_asset(InputSplatData *splats, int n, int pf, int sf, int cf, int shf, uint8_t *pos, uint8_t *other,
                                 uint8_t *col, uint8_t *sh, uint8_t *chunks, float bounds[6], uint8_t *conv_rec, uint8_t *conv_rows) {
  if (n < 1 || pf < 0 || pf > 3 || sf < 0 || sf > 3 || cf < 0 || cf > 3 || shf < 0 || shf > 8) return -1;
  int64_t sz[7];
  ref_cs_sizes(n, pf, sf, cf, shf, sz);
  NativeArray<InputSplatData> input(splats, n);

  float3 boundsMin, boundsMax;
  GaussianSplatAssetCreator::CalcBoundsJob boundsJob;
  boundsJob.m_BoundsMin = &boundsMin;
  boundsJob.m_BoundsMax = &boundsMax;
  boundsJob.m_SplatData = input;
  boundsJob.Execute();
  const float b[6] = {boundsMin.x, boundsMin.y, boundsMin.z, boundsMax.x, boundsMax.y, boundsMax.z};
  std::memcpy(bounds, b, sizeof(b));

  g_conv_events = 0;
  GaussianSplatAssetCreator::ReorderMorton(input, boundsMin, boundsMax);
  const long morton_events = g_conv_events;

  if (sz[0]) {
    GaussianSplatAssetCreator::CalcChunkDataJob job;
    job.splatData = input;
    job.chunks = NativeArray<GSA::ChunkInfo>((GSA::ChunkInfo *)chunks, (int)(sz[0] / 64));
    RunParallelFor(job, job.chunks.Length);
  }
  {
    GaussianSplatAssetCreator::CreatePositionsDataJob job;
    job.m_Input = input;
    job.m_Format = (GSA::VectorFormat)pf;
    job.m_FormatSize = GSA::GetVectorSize(job.m_Format);
    job.m_Output = NativeArray<byte>(pos, (int)sz[1]);
    run_marked(job, n, conv_rec, 1);
  }
  {
    GaussianSplatAssetCreator::CreateOtherDataJob job;
    job.m_Input = input;
    job.m_ScaleFormat = (GSA::VectorFormat)sf;
    job.m_FormatSize = GSA::GetOtherSizeNoSHIndex(job.m_ScaleFormat) + (clustered(shf) ? 2 : 0);
    job.m_Output = NativeArray<byte>(other, (int)sz[2]);
    run_marked(job, n, conv_rec, 2);
  }
  if (cf != (int)GSA::ColorFormat::BC7) {
    const int width = (int)sz[5], height = (int)sz[6];
    NativeArray<float4> data(width * height, Allocator::TempJob);
    GaussianSplatAssetCreator::CreateColorDataJob job;
    job.m_Input = input;
    job.m_Output = data;
    RunParallelFor(job, n);
    GaussianSplatAssetCreator::ConvertColorJob convert;
    convert.width = width;
    convert.height = height;
    convert.inputData = data;
    convert.format = (GSA::ColorFormat)cf;
    convert.outputData = NativeArray<byte>(col, (int)sz[3]);
    convert.formatBytesPerPixel = (int)sz[3] / width / height;
    run_marked(convert, height, conv_rows, 1);
    data.Dispose();
  }
  if (!clustered(shf)) {
    GaussianSplatAssetCreator::CreateSHDataJob job;
    job.m_Input = input;
    job.m_Format = (GSA::SHFormat)shf;
    job.m_Output = NativeArray<byte>(sh, (int)sz[4]);
    run_marked(job, n, conv_rec, 4);
  }
  return morton_events;
}

// LinearizeDataJob (E/Utils/GaussianFileReader.cs:210-233) over raw PLY-space records (rot_0..3 = w, x, y, z; log scale;
// opacity logit; f_dc), in place
REF_API void ref_cs_linearize(InputSplatData *splats, int n) {
  GaussianFileReader::LinearizeDataJob job;
  job.splatData = NativeArray<InputSplatData>(splats, n);
  RunParallelFor(job, n);
}

// The shim's stated third-party semantics, one entry each, for tests/test_reference_cs.py
REF_API uint32_t ref_cs_f32tof16(float x) { return math::f32tof16(x); }
REF_API void ref_cs_half3(const float v[3], uint16_t out[3]) {
  const half3 h(float3(v[0], v[1], v[2]));
  std::memcpy(out, &h, 6);
}
REF_API float ref_cs_pow(float x, float y) { return math::pow(x, y); }
REF_API float ref_cs_min(float x, float y) { return math::min(x, y); }
REF_API float ref_cs_max(float x, float y) { return math::max(x, y); }
REF_API float ref_cs_saturate(float x) { return math::saturate(x); }
REF_API uint32_t ref_cs_to_uint(float x, int *out_of_range) {
  g_conv_events = 0;
  const uint32_t r = conv<uint>(x);
  *out_of_range = g_conv_events ? 1 : 0;
  return r;
}
REF_API uint64_t ref_cs_to_ulong(float x, int *out_of_range) {
  g_conv_events = 0;
  const uint64_t r = conv<ulong>(x);
  *out_of_range = g_conv_events ? 1 : 0;
  return r;
}

}  // extern "C"
