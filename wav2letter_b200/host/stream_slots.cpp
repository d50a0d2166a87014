// stream_slots.cpp — the slot model shared by the streaming acoustic model (stream_capi.cpp) and its MFSC front end
// (mfsc_stream_capi.cpp): call checks, start, the per-call plan, the window kernel's arguments and the commit after a
// call.  Host arithmetic only.  DESIGN.md §4.
#include <algorithm>
#include <stdexcept>
#include <string>
#include <utility>
#include <vector>

#include "stream_internal.h"

namespace w2l {
namespace streaming {

void checkMaxStreams(const char* who, int maxStreams) {
  if (maxStreams <= 0 || maxStreams > kMaxCallStreams)
    throw std::invalid_argument(std::string(who) + "_create: max_streams must be in [1, " + std::to_string(kMaxCallStreams) + "]");
}

SlotTable::SlotTable(const char* who, int maxStreams, std::vector<ConvBuffer> buffers) : who_(who), bufs_(std::move(buffers)), slots_(maxStreams) {
  for (const ConvBuffer& b : bufs_) {
    off_.push_back(planeFloats_);
    planeFloats_ += ((long long)maxTail(b) * b.F + 3) / 4 * 4;
  }
}

void SlotTable::check(int n, const int* slots, bool forRun) const {
  const int maxStreams = (int)slots_.size();
  if (n <= 0 || n > maxStreams) throw std::invalid_argument(who_ + ": n must be in [1, max_streams]");
  if (!slots) throw std::invalid_argument(who_ + ": null slot list");
  std::vector<char> seen(maxStreams, 0);
  for (int i = 0; i < n; ++i) {
    const int k = slots[i];
    if (k < 0 || k >= maxStreams) throw std::invalid_argument(who_ + ": slot " + std::to_string(k) + " out of range [0, max_streams)");
    if (seen[k]) throw std::invalid_argument(who_ + ": slot " + std::to_string(k) + " listed twice in one call");
    seen[k] = 1;
    if (forRun && slots_[k].status == 0) throw std::invalid_argument(who_ + ": run on slot " + std::to_string(k) + ", which is not started");
    if (forRun && slots_[k].status == 2)
      throw std::invalid_argument(who_ + ": run on slot " + std::to_string(k) + ", which is finished (start it again)");
  }
}

void SlotTable::start(int n, const int* slots) {
  for (int i = 0; i < n; ++i) {
    Slot& sl = slots_[slots[i]];
    sl.status = 1;
    sl.plane = 0;
    sl.tails.clear();
    for (const ConvBuffer& b : bufs_) sl.tails.push_back(b.padL);
  }
}

Plan SlotTable::plan(int n, const int* slots, const int* framesIn, bool finish) const {
  Plan p;
  p.n = n;
  p.slots = slots;
  p.finish = finish;
  std::vector<int> cur(framesIn, framesIn + n);
  for (size_t b = 0; b < bufs_.size(); ++b) {
    const ConvBuffer& c = bufs_[b];
    std::vector<int> o(n), t(n);
    int wmax = 0, omax = 0;
    for (int i = 0; i < n; ++i) {
      const ConvStep s = convStep(slots_[slots[i]].tails[b], cur[i], finish ? c.padR : 0, c.kw, c.stride);
      o[i] = s.nOut;
      t[i] = s.tail;
      wmax = std::max(wmax, s.avail);
      omax = std::max(omax, s.nOut);
    }
    p.fresh.push_back(cur);
    p.out.push_back(o);
    p.tails.push_back(t);
    p.winFrames.push_back(wmax);
    p.outFrames.push_back(omax);
    cur = o;
  }
  p.framesOut = cur;
  p.tOutMax = n ? *std::max_element(cur.begin(), cur.end()) : 0;
  return p;
}

WindowArgs SlotTable::window(const Plan& p, size_t b, const float* in, int inFrames, float* win, int winFrames) const {
  const ConvBuffer& c = bufs_[b];
  WindowArgs a;
  a.in = in;
  a.win = win;
  a.state = state + off_[b];
  a.slotFloats = slotFloats();
  a.planeFloats = planeFloats_;
  a.inFrames = inFrames;
  a.winFrames = winFrames;
  a.F = c.F;
  a.kw = c.kw;
  a.stride = c.stride;
  a.padR = p.finish ? c.padR : 0;
  a.n = p.n;
  for (int i = 0; i < p.n; ++i) {
    const Slot& sl = slots_[p.slots[i]];
    a.code[i] = p.slots[i] << 1 | sl.plane;
    a.cnt[i] = sl.tails[b] << 16 | p.fresh[b][i];
  }
  return a;
}

void SlotTable::commit(const Plan& p, int* framesOut) {
  for (int i = 0; i < p.n; ++i) {
    Slot& sl = slots_[p.slots[i]];
    for (size_t b = 0; b < bufs_.size(); ++b) sl.tails[b] = p.tails[b][i];
    sl.plane ^= 1;
    if (p.finish) sl.status = 2;
    framesOut[i] = p.framesOut[i];
  }
}

}  // namespace streaming
}  // namespace w2l
