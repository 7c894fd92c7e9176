// key_ranges.cu -- the key-range pipeline of the keyed calls (keyed_fit.cu, k5_score.cu): the greedy range planner and the staging
// ring that brings a range's rows onto the device while the previous range runs.
#include <algorithm>
#include <chrono>
#include <cstring>
#include <string>

#include "host.cuh"

namespace mlease {

std::vector<long long> plan_ranges(long long n, size_t cap, long long limit, const std::function<size_t(long long)>& cost,
                                   const std::function<bool(long long)>& counted) {
  std::vector<long long> bounds{0};
  for (long long k = 0; k < n;) {
    long long e = k, m = 0;
    size_t bytes = 0;
    while (e < n) {
      const size_t need = cost ? cost(e) : 0;
      const bool c = !counted || counted(e);
      if (e > k && (bytes + need > cap || (c && m >= limit))) break;
      bytes += need; m += c ? 1 : 0; e++;
    }
    bounds.push_back(e);
    k = e;
  }
  return bounds;
}

void parallel_memcpy(void* dst, const void* src, size_t n) {
  const size_t per = size_t(8) << 20;
  const size_t hw = std::max(1u, std::min(8u, std::thread::hardware_concurrency()));
  const int nt = (int)std::min(hw, (n + per - 1) / per);
  if (nt <= 1) { if (n) std::memcpy(dst, src, n); return; }
  std::vector<std::thread> ts;
  const size_t step = (n + nt - 1) / nt;
  for (int t = 0; t < nt; t++) {
    const size_t a = std::min(n, t * step), b = std::min(n, a + step);
    try {
      ts.emplace_back([=] { std::memcpy((char*)dst + a, (const char*)src + a, b - a); });
    } catch (const std::exception&) {   // no thread to spare: this slice on the calling thread
      std::memcpy((char*)dst + a, (const char*)src + a, b - a);
    }
  }
  for (auto& t : ts) t.join();
}

RangeRing::~RangeRing() {
  if (stager_.joinable()) stager_.join();
  for (auto e : up_) if (e) cudaEventDestroy(e);
  for (auto e : done_) if (e) cudaEventDestroy(e);
  if (in_) cudaEventDestroy(in_);
  if (cs_) cudaStreamDestroy(cs_);
}

// the first element and the element count of source s in range c
void RangeRing::cut(const RangeSrc& s, int c, size_t* first, size_t* count) const {
  const long long r0 = row_at_[c], n = row_at_[c + 1] - r0;
  switch (s.cut) {
    case RangeSrc::ENTRY: *first = (size_t)nnz_at_[c]; *count = (size_t)(nnz_at_[c + 1] - nnz_at_[c]); break;
    case RangeSrc::ROWPTR: *first = (size_t)r0; *count = (size_t)n + 1; break;
    case RangeSrc::DENSE: *first = (size_t)(r0 * ld_); *count = n > 0 ? (size_t)((n - 1) * ld_ + Dg_) : 0; break;
    default: *first = (size_t)r0; *count = (size_t)n;
  }
}

int RangeRing::open() {
  if (!staged()) return 0;
  slot_.assign(srcs_.size(), {});
  for (size_t i = 0; i < srcs_.size(); i++) {
    const RangeSrc& s = srcs_[i];
    if (!s.p) continue;
    size_t count = 0, first, n;   // a slot holds the source's largest range
    for (int c = 0; c + 1 < (int)row_at_.size(); c++) { cut(s, c, &first, &n); count = std::max(count, n); }
    slot_[i].dma = !bounce_ || is_dma_ptr(s.p);
    for (int b = 0; b < 2; b++) {
      if (int rc = mem_.get(&slot_[i].dev[b], count * s.esize, false)) return rc;
      if (!slot_[i].dma) { if (int rc = pinned_.get(&slot_[i].host[b], count * s.esize, false)) return rc; }
    }
  }
  CK(cudaStreamCreateWithFlags(&cs_, cudaStreamNonBlocking));
  for (int b = 0; b < 2; b++) {
    CK(cudaEventCreateWithFlags(&up_[b], cudaEventDisableTiming));
    CK(cudaEventCreateWithFlags(&done_[b], cudaEventDisableTiming));
  }
  CK(cudaEventCreateWithFlags(&in_, cudaEventDisableTiming));
  CK(cudaEventRecord(in_, st_));   // device input may be produced by work the caller queued on st
  CK(cudaGetDevice(&device_));
  return start(0);
}

// range c into slot c & 1, its copies queued on cs_ and followed by up_[b]; a staging thread returns once they are done
cudaError_t RangeRing::stage(int c) {
  const int b = c & 1;
  cudaError_t e = cudaSetDevice(device_);
  if (e == cudaSuccess) e = cudaStreamWaitEvent(cs_, in_, 0);
  if (e == cudaSuccess) e = cudaStreamWaitEvent(cs_, done_[b], 0);   // range c - 2 is done with the slot (no-op before it is recorded)
  for (size_t i = 0; i < srcs_.size() && e == cudaSuccess; i++) {
    const RangeSrc& s = srcs_[i];
    if (!s.p) continue;
    size_t first, count;
    cut(s, c, &first, &count);
    const char* src = (const char*)s.p + first * s.esize;
    const size_t bytes = count * s.esize;
    if (!bytes) continue;
    if (slot_[i].dma) { e = cudaMemcpyAsync(slot_[i].dev[b], src, bytes, cudaMemcpyDefault, cs_); continue; }
    parallel_memcpy(slot_[i].host[b], src, bytes);
    e = cudaMemcpyAsync(slot_[i].dev[b], slot_[i].host[b], bytes, cudaMemcpyHostToDevice, cs_);
  }
  if (e == cudaSuccess) e = cudaEventRecord(up_[b], cs_);
  if (e == cudaSuccess && bounce_) e = cudaEventSynchronize(up_[b]);   // the pinned buffer is reused two ranges on
  return e;
}

int RangeRing::start(int c) {
  if (!staged() || c + 1 >= (int)row_at_.size()) return 0;
  auto run = [this, c] {
    const auto t0 = std::chrono::steady_clock::now();
    stage_err_ = stage(c);
    stage_ms += std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
  };
  if (!bounce_) { run(); return 0; }   // direct copies, queued: the copy engines overlap them with the running range
  try {
    stager_ = std::thread(run);
  } catch (const std::exception& e) {   // no exception leaves the C ABI
    return fail(MLEASE_ERR_CUDA, std::string("cannot start the staging thread: ") + e.what());
  }
  return 0;
}

int RangeRing::view(int c, const void** v) {
  if (!staged()) {
    for (size_t i = 0; i < srcs_.size(); i++) v[i] = srcs_[i].p;
    return 0;
  }
  const auto t0 = std::chrono::steady_clock::now();
  if (stager_.joinable()) stager_.join();
  wait_ms += std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
  if (stage_err_ != cudaSuccess) return fail(MLEASE_ERR_CUDA, std::string("staging the rows of a key range: ") + cudaGetErrorString(stage_err_));
  CK(cudaStreamWaitEvent(st_, up_[c & 1], 0));
  for (size_t i = 0; i < srcs_.size(); i++) v[i] = srcs_[i].p ? slot_[i].dev[c & 1] : nullptr;
  return 0;
}

int RangeRing::done(int c) {
  if (staged()) CK(cudaEventRecord(done_[c & 1], st_));
  return 0;
}

}  // namespace mlease
