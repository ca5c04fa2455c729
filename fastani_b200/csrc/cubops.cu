// cubops.cu -- the device-wide primitives taken from CUB (radix sort, exclusive scan).
// Kept in one translation unit because CUB instantiations dominate compile time.
// These are library calls (like cuBLAS would be for a GEMM); the kernels specific to the
// ANI hot path live in sketch.cu / index.cu / map.cu.
#include <cub/cub.cuh>
#include "common.cuh"

namespace bani {

size_t cub_sort_pairs_u32_temp(size_t n)
{
  size_t b = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, b, (const uint32_t *)nullptr, (uint32_t *)nullptr,
                                  (const uint32_t *)nullptr, (uint32_t *)nullptr, n);
  return b;
}
void cub_sort_pairs_u32(void *temp, size_t tempBytes, const uint32_t *kin, uint32_t *kout,
                        const uint32_t *vin, uint32_t *vout, size_t n, int endBit, cudaStream_t s)
{
  BANI_CUDA(cub::DeviceRadixSort::SortPairs(temp, tempBytes, kin, kout, vin, vout, n, 0, endBit, s));
}
size_t cub_sort_keys_u64_temp(size_t n)
{
  size_t b = 0;
  cub::DeviceRadixSort::SortKeys(nullptr, b, (const uint64_t *)nullptr, (uint64_t *)nullptr, n);
  return b;
}
void cub_sort_keys_u64(void *temp, size_t tempBytes, const uint64_t *kin, uint64_t *kout, size_t n,
                       int beginBit, int endBit, cudaStream_t s)
{
  BANI_CUDA(cub::DeviceRadixSort::SortKeys(temp, tempBytes, kin, kout, n, beginBit, endBit, s));
}
size_t cub_sort_pairs_u64_u32_temp(size_t n)
{
  size_t b = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, b, (const uint64_t *)nullptr, (uint64_t *)nullptr,
                                  (const uint32_t *)nullptr, (uint32_t *)nullptr, n);
  return b;
}
void cub_sort_pairs_u64_u32(void *temp, size_t tempBytes, const uint64_t *kin, uint64_t *kout,
                            const uint32_t *vin, uint32_t *vout, size_t n, int endBit, cudaStream_t s)
{
  BANI_CUDA(cub::DeviceRadixSort::SortPairs(temp, tempBytes, kin, kout, vin, vout, n, 0, endBit, s));
}
size_t cub_scan_u32_temp(size_t n)
{
  size_t b = 0;
  cub::DeviceScan::ExclusiveSum(nullptr, b, (const uint32_t *)nullptr, (uint32_t *)nullptr, n);
  return b;
}
void cub_exclusive_sum_u32(void *temp, size_t tempBytes, const uint32_t *in, uint32_t *out, size_t n, cudaStream_t s)
{
  BANI_CUDA(cub::DeviceScan::ExclusiveSum(temp, tempBytes, in, out, n, s));
}
struct U32toU64 { __host__ __device__ uint64_t operator()(uint32_t x) const { return (uint64_t)x; } };
size_t cub_scan_u64_temp(size_t n)
{
  size_t b = 0;
  cub::TransformInputIterator<uint64_t, U32toU64, const uint32_t *> it((const uint32_t *)nullptr, U32toU64());
  cub::DeviceScan::ExclusiveSum(nullptr, b, it, (uint64_t *)nullptr, n);
  return b;
}
void cub_exclusive_sum_u32_to_u64(void *temp, size_t tempBytes, const uint32_t *in, uint64_t *out, size_t n, cudaStream_t s)
{
  cub::TransformInputIterator<uint64_t, U32toU64, const uint32_t *> it(in, U32toU64());
  BANI_CUDA(cub::DeviceScan::ExclusiveSum(temp, tempBytes, it, out, n, s));
}

} // namespace bani
