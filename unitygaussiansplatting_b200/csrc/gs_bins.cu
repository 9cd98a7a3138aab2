// gs_bins.cu -- the bin list's CUDA calls (BinList, gs_internal.cuh): its buffers grown and its entry counts read back.
#include "gs_internal.cuh"

namespace gs {

int BinList::reserve(GsContext *ctx, uint32_t n, uint32_t bins, uint32_t min_capacity) {
  const uint32_t want = std::max(capacity_for(n), min_capacity);
  GS_CUDA_TRY(ctx, keys.reserve(want, {ctx->stream}));
  GS_CUDA_TRY(ctx, vals.reserve(want, {ctx->stream}));
  const int rc = ensure_sort_scratch(ctx, std::max(capacity(), n));
  if (rc) return rc;
  const uint32_t blocks = n / 1024 + 2 < 1024u ? 1024u : n / 1024 + 2;   // the binner's ticket + range totals (<= 593 words) fit too
  GS_CUDA_TRY(ctx, block_sums.reserve(blocks, {ctx->stream}));
  GS_CUDA_TRY(ctx, ranges.reserve(bins, {ctx->stream}));
  return GS_OK;
}

cudaError_t BinList::read(GsContext *ctx, uint32_t *ec, uint32_t words) {
  const cudaError_t e = cudaMemcpyAsync(ec, entry_count.get(), words * 4, cudaMemcpyDeviceToHost, ctx->stream);
  return e != cudaSuccess ? e : cudaStreamSynchronize(ctx->stream);
}

uint32_t BinList::capacity() const { return (uint32_t)std::min(keys.size(), vals.size()); }

int BinList::check(GsContext *ctx) {
  uint32_t ec[2] = {0, 0};
  GS_CUDA_TRY(ctx, read(ctx, ec, 2));
  ctx->times.tile_entries = ec[0];
  if (ec[1]) return fail(ctx, GS_ERR_OUT_OF_MEMORY, "tile-list capacity exceeded (splat footprints cover too many tiles)");
  return GS_OK;
}

}  // namespace gs
