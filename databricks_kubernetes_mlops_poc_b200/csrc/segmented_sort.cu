/*
 * segmented_sort.cu -- the per-point sort of K8 (permutation_importance.cuh): CUB's segmented radix sort of
 * (ranking key, flags) pairs, stable and deterministic.  It is a translation unit of its own so that CUB's device
 * globals live in their own module: the kernels of b2f_api.cu keep their constant-bank layout.
 */
#include <cub/device/device_segmented_radix_sort.cuh>
#include <stdint.h>

/* Sort each of `segs` segments [off[s], off[s + 1]) of the double buffers (k0, f0) / (k1, f1) by the 64-bit key.  With
 * temp == NULL: the temporary bytes needed, in *temp_bytes.  *current: 0 when the result is in (k0, f0), 1 in (k1, f1). */
cudaError_t pi_segmented_sort(void *temp, size_t *temp_bytes, unsigned long long *k0, unsigned long long *k1, uint8_t *f0, uint8_t *f1,
                              int items, int segs, const int *off, cudaStream_t st, int *current) {
    cub::DoubleBuffer<unsigned long long> dk(k0, k1);
    cub::DoubleBuffer<uint8_t> dv(f0, f1);
    const cudaError_t e = cub::DeviceSegmentedRadixSort::SortPairs(temp, *temp_bytes, dk, dv, items, segs, off, off + 1, 0, 64, st);
    if (current) *current = dk.selector;
    return e;
}
