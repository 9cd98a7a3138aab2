// asset_cluster_bc7.cpp -- the two lossy stages of the importer's VeryLow / Low presets (libgsplat_asset.so):
//   * SH palette clustering: mini-batch k-means with k-means++ seeding, following the reference's algorithm step by step
//     (package/Editor/Utils/KMeansClustering.cs, cited below as K:line) so that the same input yields the same palette:
//     same RNG (pcg, state 1), same batch draws, same sequential centroid update, same summation order in the squared
//     distance (the x86 AVX path of K:144-167: eight squares, pairwise add, then left-to-right).
//     New code: one flat implementation with the candidate means laid out dimension-major so that eight / sixteen
//     distances are evaluated side by side (each lane keeps the scalar operation order, so results equal the scalar ones).
//   * BC7 colour: the reference calls Unity's closed-source texture compressor (E/GaussianSplatAssetCreator.cs:901-912),
//     which cannot be reproduced; any conformant BC7 stream decodes the same way on the GPU, so this packer emits mode-6
//     blocks (one subset, 7.7.7.7 endpoints + p-bits, 4-bit indices) from a principal-axis fit.  Lossy, NOT bit-identical
//     to Unity's encoder; the decode side (gs_bc7.cuh / oracle) handles all eight modes.
// The pcg stream, the batch draw, the squared distance and the BC7 block encoder are gs_asset_format.h, shared with the
// GPU packer (gs_pack.cu).
#include "../../include/gsplat_asset.h"
#include "gs_asset_format.h"

#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <limits>
#include <cstdio>
#include <cstdlib>
#include <vector>
#ifdef __linux__
#include <sched.h>
#endif
#ifdef _OPENMP
#include <omp.h>
#endif

namespace {

// Threads worth starting: OpenMP's default, but never more than the CPUs this process may actually use -- its affinity mask
// and its cgroup CPU quota (a container can show 64 cores and be allowed 8; spinning at barriers then eats the quota).
int usable_threads_uncached() {
  int t = 1;
#ifdef _OPENMP
  t = omp_get_max_threads();
#endif
#ifdef __linux__
  cpu_set_t set;
  if (sched_getaffinity(0, sizeof(set), &set) == 0) t = std::min(t, std::max(1, CPU_COUNT(&set)));
  long long quota = -1, period = -1;
  if (FILE *f = std::fopen("/sys/fs/cgroup/cpu.max", "r")) {            // cgroup v2: "<quota|max> <period>"
    char q[32];
    if (std::fscanf(f, "%31s %lld", q, &period) == 2 && std::strcmp(q, "max") != 0) quota = std::atoll(q);
    std::fclose(f);
  } else {                                                              // cgroup v1
    if (FILE *g = std::fopen("/sys/fs/cgroup/cpu/cpu.cfs_quota_us", "r")) { if (std::fscanf(g, "%lld", &quota) != 1) quota = -1; std::fclose(g); }
    if (FILE *g = std::fopen("/sys/fs/cgroup/cpu/cpu.cfs_period_us", "r")) { if (std::fscanf(g, "%lld", &period) != 1) period = -1; std::fclose(g); }
  }
  if (quota > 0 && period > 0) t = std::min<long long>(t, std::max<long long>(1, (quota + period - 1) / period));
#endif
  return std::max(1, t);
}
int usable_threads() { static const int t = usable_threads_uncached(); return t; }
// the k-means++ and mini-batch phases alternate short parallel loops with serial steps thousands of times: a small team
// keeps the fork/join and barrier cost below the work (each loop is 1-5 ms of arithmetic)
inline int small_team(int threads) { return std::min(threads, 16); }

using namespace gs;

// The same arithmetic for L candidate means at once.  `mt` is dimension-major: mt[c * stride + j] = means[j][c].
template <int L>
inline void distance_squared_lanes(int dim, const float *a, const float *mt, size_t stride, float *out) {
  float d[L];
  for (int l = 0; l < L; ++l) d[l] = 0;
  int i = 0;
  for (; i + 7 < dim; i += 8) {
    float h[4][L];
    for (int p = 0; p < 4; ++p) {
      const float a0 = a[i + 2 * p], a1 = a[i + 2 * p + 1];
      const float *m0 = mt + (size_t)(i + 2 * p) * stride, *m1 = m0 + stride;
      for (int l = 0; l < L; ++l) {
        float t0 = a0 - m0[l], t1 = a1 - m1[l];
        h[p][l] = t0 * t0 + t1 * t1;
      }
    }
    for (int l = 0; l < L; ++l) d[l] += ((h[0][l] + h[1][l]) + h[2][l]) + h[3][l];
  }
  for (; i < dim; ++i) {
    const float ai = a[i];
    const float *m = mt + (size_t)i * stride;
    for (int l = 0; l < L; ++l) { float t = ai - m[l]; d[l] += t * t; }
  }
  for (int l = 0; l < L; ++l) out[l] = d[l];
}

struct MeansT {  // dimension-major copy of k means, padded to a multiple of 16 with +inf-distance dummies
  int dim = 0, k = 0;
  size_t stride = 0;
  std::vector<float> t;
  void build(int dim_, int k_, const float *means) {
    dim = dim_; k = k_;
    stride = ((size_t)k + 15) / 16 * 16;
    t.assign((size_t)dim * stride, 0.0f);
    for (int j = 0; j < k; ++j)
      for (int c = 0; c < dim; ++c) t[(size_t)c * stride + j] = means[(size_t)j * dim + c];
  }
  void set(int j, const float *mean) {
    for (int c = 0; c < dim; ++c) t[(size_t)c * stride + j] = mean[c];
  }
};

// AssignClustersJob.Execute, K:423-441: nearest mean, first one wins ties (strict <)
inline int nearest_mean(const MeansT &m, const float *p, float *min_dist_out) {
  float best = std::numeric_limits<float>::max();
  int best_i = 0;
  float d[16];
  for (int j = 0; j < m.k; j += 16) {
    distance_squared_lanes<16>(m.dim, p, m.t.data() + j, m.stride, d);
    const int lim = std::min(16, m.k - j);
    for (int l = 0; l < lim; ++l)
      if (d[l] < best) { best = d[l]; best_i = j + l; }
  }
  if (min_dist_out) *min_dist_out = best;
  return best_i;
}

// MakeBatchJob, K:456-477: distinct random points in draw order
void make_random_batch(int dim, const float *data, uint32_t data_size, uint32_t &rng, float *out, uint32_t batch,
                       std::vector<uint8_t> &picked) {
  std::vector<uint32_t> chosen(batch);
  random_batch(data_size, rng, batch, picked.data(), chosen.data());
  for (uint32_t i = 0; i < batch; ++i) std::memcpy(out + (size_t)i * dim, data + (size_t)chosen[i] * dim, (size_t)dim * 4);
}

// KMeansPlusPlus, K:325-411 (+ PickPointIndex K:273-323, CalcDistSqJob K:249-271)
void kmeans_plus_plus(int dim, int k, const float *data, uint32_t data_size, float *means, float *min_dist_sq, uint32_t &rng, int threads) {
  const int team = small_team(threads);
  (void)team;
  std::vector<uint8_t> taken(data_size, 0);
  int point = (int)(pcg_random(rng) % data_size);
  taken[point] = 1;
  std::memcpy(means, data + (size_t)point * dim, (size_t)dim * 4);
#pragma omp parallel for schedule(static) num_threads(team)
  for (int64_t i = 0; i < (int64_t)data_size; ++i)
    if (i != point) min_dist_sq[i] = distance_squared(data + (size_t)i * dim, means, dim);
  constexpr int kSumBatch = 1024;
  const int sum_batches = (int)((data_size + kSumBatch - 1) / kSumBatch);
  std::vector<float> partial(sum_batches);
  int result_count = 1;
  const float *new_mean = nullptr;   // centre picked in the previous round: its distance update rides in this round's loop
  while (result_count < k) {
    // ClosestDistanceUpdateJob (K:235-247) for the newest centre, then CalcDistSqJob (K:249-271): one pass per 1024-point
    // batch, element order inside a batch as in the reference, so sums are the same floats
#pragma omp parallel for schedule(static) num_threads(team)
    for (int b = 0; b < sum_batches; ++b) {
      const uint32_t i0 = std::min<uint32_t>((uint32_t)b * kSumBatch, data_size), i1 = std::min<uint32_t>((uint32_t)(b + 1) * kSumBatch, data_size);
      float sum = 0;
      for (uint32_t i = i0; i < i1; ++i) {
        if (taken[i]) continue;
        if (new_mean) min_dist_sq[i] = std::min(min_dist_sq[i], distance_squared(data + (size_t)i * dim, new_mean, dim));
        sum += min_dist_sq[i];
      }
      partial[b] = sum;
    }
    float total = 0;
    for (int b = 0; b < sum_batches; ++b) { total += partial[b]; partial[b] = total; }
    const float rval = pcg_hash_float(rng + (uint32_t)result_count, total);
    // PickPointIndex
    int lo = 0, hi = sum_batches;
    while (lo < hi) {
      int mid = (lo + hi) / 2;
      if (partial[mid] < rval) lo = mid + 1; else hi = mid;
    }
    float acc = lo > 0 ? partial[lo - 1] : 0.0f;
    point = -1;
    for (uint32_t i = (uint32_t)lo * kSumBatch; i < data_size; ++i) {
      if (taken[i]) continue;
      acc += min_dist_sq[i];
      if (acc >= rval) { point = (int)i; break; }
    }
    if (point < 0)
      for (int64_t i = (int64_t)data_size - 1; i >= 0; --i)
        if (!taken[i]) { point = (int)i; break; }
    if (point < 0) point = 0;
    taken[point] = 1;
    float *slot = means + (size_t)result_count * dim;
    std::memcpy(slot, data + (size_t)point * dim, (size_t)dim * 4);
    new_mean = slot;
    ++result_count;
  }
}

// InitializeCentroids, K:507-569
void initialize_centroids(int dim, const float *data, uint32_t data_size, uint32_t init_batch, uint32_t &rng, int attempts, float *out_means,
                          int k, std::vector<uint8_t> &picked, int threads) {
  init_batch = std::min(init_batch, data_size);
  std::vector<float> centroid_batch((size_t)init_batch * dim), validation_batch((size_t)init_batch * dim);
  make_random_batch(dim, data, data_size, rng, centroid_batch.data(), init_batch, picked);
  make_random_batch(dim, data, data_size, rng, validation_batch.data(), init_batch, picked);
  std::vector<float> tmp_dist(init_batch, 0.0f), cur((size_t)k * dim);
  float min_dist_sum = std::numeric_limits<float>::max();
  MeansT mt;
  for (int ia = 0; ia < attempts; ++ia) {
    kmeans_plus_plus(dim, k, centroid_batch.data(), init_batch, cur.data(), tmp_dist.data(), rng, threads);
    mt.build(dim, k, cur.data());
#pragma omp parallel for schedule(dynamic, 64) num_threads(threads)
    for (int64_t i = 0; i < (int64_t)init_batch; ++i) nearest_mean(mt, validation_batch.data() + (size_t)i * dim, &tmp_dist[i]);
    float dist_sum = 0;
    for (uint32_t i = 0; i < init_batch; ++i) dist_sum += tmp_dist[i];
    if (dist_sum < min_dist_sum) {
      min_dist_sum = dist_sum;
      std::memcpy(out_means, cur.data(), (size_t)k * dim * 4);
    }
  }
}

}  // namespace

int gsa_usable_threads() { return usable_threads(); }

extern "C" {

// KMeansClustering.Calculate, K:29-136
int gsa_kmeans(uint32_t dim, const float *data, uint32_t data_size, uint32_t batch_size, float passes_over_data, float *out_means, uint32_t k,
               int32_t *out_labels) {
  if (!data || !out_means || !out_labels || dim < 1 || batch_size < 1 || passes_over_data < 0.0001f || k < 1 || data_size < k) return -1;
  batch_size = std::min(data_size, batch_size);
  uint32_t rng = 1;
  std::vector<uint8_t> picked(data_size, 0);
  const int threads = usable_threads(), team = small_team(threads);
  initialize_centroids((int)dim, data, data_size, 10u * k, rng, 3, out_means, (int)k, picked, threads);

  std::vector<float> counts(k, 0.0f), batch_points((size_t)batch_size * dim);
  std::vector<int> batch_clusters(batch_size);
  MeansT mt;
  mt.build((int)dim, (int)k, out_means);
  const float calc_limit = (float)data_size * passes_over_data;
  for (float calc_done = 0.0f; calc_done < calc_limit; calc_done += (float)batch_size) {
    make_random_batch((int)dim, data, data_size, rng, batch_points.data(), batch_size, picked);
#pragma omp parallel for schedule(dynamic, 16) num_threads(team)
    for (int64_t i = 0; i < (int64_t)batch_size; ++i) batch_clusters[i] = nearest_mean(mt, batch_points.data() + (size_t)i * dim, nullptr);
    // UpdateCentroidsJob, K:479-505: strictly sequential, per-centre learning rate 1/count
    for (uint32_t i = 0; i < batch_size; ++i) {
      const int c = batch_clusters[i];
      counts[c] += 1.0f;
      const float alpha = 1.0f / counts[c];
      float *m = out_means + (size_t)c * dim;
      const float *p = batch_points.data() + (size_t)i * dim;
      for (uint32_t j = 0; j < dim; ++j) m[j] = m[j] + alpha * (p[j] - m[j]);  // math.lerp(x, y, s) = x + s * (y - x)
    }
    for (uint32_t i = 0; i < batch_size; ++i) mt.set(batch_clusters[i], out_means + (size_t)batch_clusters[i] * dim);
  }
#pragma omp parallel for schedule(dynamic, 256) num_threads(threads)
  for (int64_t i = 0; i < (int64_t)data_size; ++i) out_labels[i] = nearest_mean(mt, data + (size_t)i * dim, nullptr);
  return 0;
}

// One 4x4 block of float RGBA in [0,1] (raster order) -> 16 bytes of BC7 mode 6.
void gsa_bc7_encode_block(const float rgba[64], uint8_t out[16]) {
  const Bc7Block b = bc7_encode_block(rgba);
  std::memcpy(out, &b.lo, 8);
  std::memcpy(out + 8, &b.hi, 8);
}

}  // extern "C"
