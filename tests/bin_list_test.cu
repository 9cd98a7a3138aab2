// gs::BinList's rules (csrc/gs_internal.cuh) on their own, without a device: the capacity rule, the growth of a list on a
// large screen, and which build of a public call clears the overflow flag (DESIGN.md, "Overflow across a call").  The rules'
// own begin_draw / end_draw run against a model of the list on the device, which stands in for BinList's out-of-line methods
// (gs_bins.cu: the buffers and the CUDA calls).
#include <cstdint>
#include <cstdio>

#include "gs_internal.cuh"

using gs::BinList;

#define CHECK(cond)                                                     \
  do {                                                                  \
    if (!(cond)) {                                                      \
      std::printf("bin_list_test:%d: check failed: %s\n", __LINE__, #cond); \
      return 1;                                                         \
    }                                                                   \
  } while (0)

constexpr uint32_t kMi = 1u << 20;

// The list on the device: its capacity and entry_count = [clamped count, overflow flag, total].  A build clears the flag or only
// ever sets it, then sets it when the total exceeds the capacity (k_bin_emit).
static struct Device {
  uint32_t capacity = 4 * kMi, ec[3] = {0, 0, 0};
  int reads = 0;   // read-backs so far
  void build(bool clear, uint32_t total) {
    ec[1] = (clear ? 0u : ec[1]) | (total > capacity ? 1u : 0u);
    ec[0] = total > capacity ? capacity : total;
    ec[2] = total;
  }
} dev;

namespace gs {
cudaError_t BinList::read(GsContext *, uint32_t *ec, uint32_t words) {
  ++dev.reads;
  for (uint32_t i = 0; i < words; ++i) ec[i] = dev.ec[i];
  return cudaSuccess;
}
int BinList::reserve(GsContext *, uint32_t n, uint32_t, uint32_t min_capacity) {   // a buffer only ever grows
  dev.capacity = std::max(dev.capacity, std::max(capacity_for(n), min_capacity));
  return GS_OK;
}
uint32_t BinList::capacity() const { return dev.capacity; }
int fail_cuda(GsContext *, cudaError_t, const char *, const char *, int) { return GS_ERR_CUDA; }
}  // namespace gs

// What one draw did: whether it read the flag back before it started, the clear flag of its builds, what it grew the list to,
// and how many read-backs it made in all.
struct Draw {
  bool ok = true, pre_read = false, first_clears = false, rebuilt = false, rebuild_clears = false;
  uint32_t grown_to = 0;
  int reads = 0;
};

// One draw of `cameras` cameras on a screen of bins_x x bins_y bins whose list holds `total` entries, as do_draw and draw_run
// drive it.  A run of one pair begins its draw twice (draw_run, then do_draw): the second begin must read nothing.
static Draw draw(BinList &b, uint32_t cameras, uint32_t bins_x, uint32_t bins_y, uint32_t total) {
  gs::FrameConsts fc{};
  fc.binsX = bins_x;
  fc.binsY = bins_y;
  Draw d;
  const int reads = dev.reads;
  d.ok = b.begin_draw(nullptr, cameras, fc) == GS_OK;
  d.pre_read = dev.reads > reads;
  d.ok &= b.begin_draw(nullptr, cameras, fc) == GS_OK && dev.reads == reads + (d.pre_read ? 1 : 0);
  d.first_clears = b.clears();
  dev.build(d.first_clears, total);
  d.ok &= b.end_draw(nullptr, 0, bins_x * bins_y, &d.rebuilt, &d.rebuild_clears) == GS_OK;
  if (d.rebuilt) {
    d.grown_to = dev.capacity;
    dev.build(d.rebuild_clears, total);
  }
  d.reads = dev.reads - reads;
  return d;
}

static int capacity_rule() {
  CHECK(BinList::capacity_for(0) == 4 * kMi);
  CHECK(BinList::capacity_for(512 * 1024) == 4 * kMi);
  CHECK(BinList::capacity_for(512 * 1024 + 1) == 4 * kMi + 8);
  CHECK(BinList::capacity_for(96 * kMi) == 768 * kMi);
  CHECK(BinList::capacity_for(96 * kMi + 1) == 768 * kMi);
  CHECK(BinList::capacity_for(UINT32_MAX) == 768 * kMi);
  CHECK(gs::kBinListMax == 768 * kMi);
  return 0;
}

static int growth() {
  const uint32_t big = gs::kRuleBins + 1;
  BinList b;
  struct Case { uint32_t capacity, total, grown_to; } cases[] = {
    {4 * kMi, 4 * kMi, 0},                                        // fits
    {4 * kMi, 4 * kMi + 1, 4 * kMi + 1 + (4 * kMi + 1) / 4},      // total plus a quarter
    {49 * kMi, 101 * kMi, 101 * kMi + 101 * kMi / 4},
    {4 * kMi, 700 * kMi, 768 * kMi},                              // capped
    {4 * kMi, 768 * kMi, 768 * kMi},
    {4 * kMi, 768 * kMi + 1, 0},                                  // no list holds it: left truncated
    {4 * kMi, UINT32_MAX, 0},
  };
  for (const Case &c : cases) {
    b.begin_call();
    dev.capacity = c.capacity;
    const Draw d = draw(b, 1, big, 1, c.total);
    CHECK(d.ok && d.reads == 1 && d.rebuilt == (c.grown_to != 0) && d.grown_to == c.grown_to);
    CHECK(dev.ec[1] == (c.total > dev.capacity ? 1u : 0u));   // a grown list is complete, a list above 768 Mi is not
  }
  // which draws read their list back: one camera above 128 bins on either axis
  b.begin_call();
  dev.capacity = 4 * kMi;
  CHECK(draw(b, 1, gs::kRuleBins, gs::kRuleBins, 5 * kMi).reads == 0);   // 8160 x 8160 px
  CHECK(draw(b, 2, big, big, kMi).reads == 0);                          // a run of two cameras
  CHECK(draw(b, 1, 1, big, kMi).reads == 2);                            // the flag first, then the list
  CHECK(draw(b, 1, big, 1, kMi).reads == 1);
  return 0;
}

static int calls() {
  const uint32_t big = 200, small = 30;   // bins per axis: a 12800 px and a 1920 px screen
  BinList b;
  dev = Device{};
  // A draw that reads back but whose total no list holds: left truncated, and nothing is built again.
  b.begin_call();
  Draw d = draw(b, 1, big, big, 800 * kMi);
  CHECK(d.ok && !d.pre_read && d.first_clears && !d.rebuilt && dev.ec[1]);

  // A new call: its first draw grows its list, and the rebuild clears the flag the earlier call left.  A second growing draw
  // of the call, after a rebuild that cleared the flag, clears it again.
  b.begin_call();
  d = draw(b, 1, big, big, 5 * kMi);
  CHECK(d.ok && !d.pre_read && d.first_clears && d.rebuilt && d.rebuild_clears && d.grown_to == 5 * kMi + 5 * kMi / 4 && !dev.ec[1]);
  d = draw(b, 1, big, big, 8 * kMi);
  CHECK(d.ok && !d.pre_read && !d.first_clears && d.rebuilt && d.rebuild_clears && !dev.ec[1]);

  // A truncated first draw (a small screen: not read back), then a growing draw that fits: the flag is read first, and the
  // grown list keeps it set, so the call still reports the first draw.
  b.begin_call();
  dev.capacity = 4 * kMi;
  d = draw(b, 1, small, small, 5 * kMi);
  CHECK(d.ok && !d.pre_read && d.first_clears && !d.rebuilt && dev.ec[1]);
  d = draw(b, 1, big, big, 6 * kMi);
  CHECK(d.ok && d.pre_read && !d.first_clears && d.rebuilt && !d.rebuild_clears && dev.capacity == 6 * kMi + 6 * kMi / 4 && dev.ec[1]);
  // and a later growing draw of the same call needs no read: the last draw read the list back
  d = draw(b, 1, big, big, 9 * kMi);
  CHECK(d.ok && !d.pre_read && d.rebuilt && !d.rebuild_clears && dev.ec[1]);

  // A call whose draws fit until a read-back draw is truncated beyond any list: a later growing draw keeps the flag set.
  b.begin_call();
  d = draw(b, 1, big, big, kMi);
  CHECK(d.ok && d.first_clears && !d.rebuilt && !dev.ec[1]);
  d = draw(b, 1, big, big, 900 * kMi);
  CHECK(d.ok && !d.pre_read && !d.first_clears && !d.rebuilt && dev.ec[1]);
  d = draw(b, 1, big, big, 20 * kMi);
  CHECK(d.ok && !d.pre_read && d.rebuilt && !d.rebuild_clears && dev.ec[1]);

  // A growing draw after one that did not read back (a run of two cameras) and fit: the flag is read first.  The state the
  // last call left (truncated) must not keep the flag set.
  b.begin_call();
  d = draw(b, 2, small, small, kMi);
  CHECK(d.ok && d.first_clears && !d.rebuilt && !dev.ec[1]);
  d = draw(b, 1, big, big, 40 * kMi);
  CHECK(d.ok && d.pre_read && !d.first_clears && d.rebuilt && d.rebuild_clears && !dev.ec[1]);
  // and a small draw after it: nothing to read, its build only ever sets the flag
  d = draw(b, 1, small, small, kMi);
  CHECK(d.ok && !d.pre_read && !d.first_clears && !d.rebuilt && d.reads == 0 && !dev.ec[1]);
  return 0;
}

int main() {
  int rc = 0;
  if ((rc = capacity_rule()) || (rc = growth()) || (rc = calls())) return rc;
  std::printf("bin_list_test: ok\n");
  return 0;
}
