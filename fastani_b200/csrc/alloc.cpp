// alloc.cpp -- caching device allocator behind DevBuf.
//
// The hot path re-creates the same multi-GB buffers every step (index arrays, sort scratch).  Going to
// the driver for them (cudaMalloc / cudaMallocAsync + pool trimming) costs up to hundreds of milliseconds
// and is not repeatable, so freed blocks are kept per (device, stream, size) and handed out again; the
// driver is only asked on a miss, and everything cached is returned to it when an allocation fails or
// when the last context of the device goes away.  Reuse is stream-ordered: a block is only ever reused
// on the stream it was freed on, so no event is needed.
#include <algorithm>
#include <atomic>
#include <map>
#include <mutex>
#include <tuple>
#include "common.cuh"

namespace bani {

namespace {
struct Key {
  int dev; cudaStream_t st; size_t bytes;
  bool operator<(const Key &o) const { return std::tie(dev, st, bytes) < std::tie(o.dev, o.st, o.bytes); }
};
std::mutex g_mu;
std::multimap<Key, void *> g_free;
// per device: bytes handed out and not yet freed, bytes held in the cache, and the high-water mark of the former
struct Usage { size_t live = 0, cached = 0, peak = 0; };
std::map<int, Usage> g_use;

void note_live(int dev, size_t b)           // g_mu held
{
  Usage &u = g_use[dev];
  u.live += b;
  u.peak = std::max(u.peak, u.live);
}
}

// the size a request is rounded to (and cached under); index_footprint counts buffers with it
size_t dev_round_size(size_t b)
{
  if (b <= 4096) return (b + 255) & ~(size_t)255;
  if (b <= (1u << 20)) return (b + 4095) & ~(size_t)4095;
  return (b + ((size_t)2 << 20) - 1) & ~(((size_t)2 << 20) - 1);
}

uint64_t next_genome_uid()
{
  static std::atomic<uint64_t> n(1);
  return n++;
}

void dev_cache_flush(int dev)
{
  std::lock_guard<std::mutex> lk(g_mu);
  for (auto it = g_free.begin(); it != g_free.end();) {
    if (dev < 0 || it->first.dev == dev) { g_use[it->first.dev].cached -= it->first.bytes; cudaFree(it->second); it = g_free.erase(it); }
    else ++it;
  }
}

void *dev_alloc(size_t bytes, cudaStream_t st, size_t *granted, int *devOut)
{
  int dev = 0; cudaGetDevice(&dev);
  *devOut = dev;
  const size_t rb = dev_round_size(bytes);
  *granted = rb;
  {
    std::lock_guard<std::mutex> lk(g_mu);
    auto it = g_free.find(Key{dev, st, rb});
    if (it != g_free.end()) { void *p = it->second; g_free.erase(it); g_use[dev].cached -= rb; note_live(dev, rb); return p; }
  }
  void *p = nullptr;
  cudaError_t e = cudaMalloc(&p, rb);
  if (e != cudaSuccess) {
    (void)cudaGetLastError();
    cudaDeviceSynchronize();
    dev_cache_flush(dev);
    e = cudaMalloc(&p, rb);
    if (e != cudaSuccess) { (void)cudaGetLastError(); fail(BANI_ERR_NOMEM, "device allocation of %zu bytes failed: %s", rb, cudaGetErrorString(e)); }
  }
  std::lock_guard<std::mutex> lk(g_mu);
  note_live(dev, rb);
  return p;
}

void dev_free(void *p, size_t granted, cudaStream_t st, int dev)
{
  if (!p) return;
  // keyed by the device the block was ALLOCATED on (recorded in DevBuf), not by the caller's current device: a host
  // thread that drives several GPUs may destroy an object of device A while device B is current
  std::lock_guard<std::mutex> lk(g_mu);
  g_free.emplace(Key{dev, st, granted}, p);
  Usage &u = g_use[dev];
  u.live -= granted; u.cached += granted;
}

void dev_mem_stats(int dev, size_t *live, size_t *cached, size_t *peak)
{
  std::lock_guard<std::mutex> lk(g_mu);
  const Usage &u = g_use[dev];
  if (live) *live = u.live;
  if (cached) *cached = u.cached;
  if (peak) *peak = u.peak;
}

void dev_mem_peak_set(int dev, size_t v)
{
  std::lock_guard<std::mutex> lk(g_mu);
  Usage &u = g_use[dev];
  u.peak = std::max(v, u.live);
}

} // namespace bani
