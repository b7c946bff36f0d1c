// gsplat's intersection keys and tile offsets for one camera (the gsplat-v1 drop-in's isect_tiles / isect_offset_encode).
//
// The hierarchical binning (binning.cu) produces per-tile id lists and never materialises gsplat's 64-bit keys.  Their order
// equals a stable sort of (tile << 32 | float_bits(depth)) keys, so the keys of our list order are gsplat's sorted isect_ids:
// one pass over tile_ranges / sorted_ids rebuilds them.  The offsets are a binary search per tile over whatever sorted keys
// the caller hands over, so they never depend on the binning's state.
#include "common.cuh"

namespace b200gs {

namespace {

constexpr int KEYS_THREADS = 256;   // one warp per tile: 8 tiles per block
constexpr int OFFSETS_THREADS = 256;

// keys[i] = (tile << 32) | float_bits(depth[sorted_ids[i]]) for every listed pair i of every tile.  The lanes of a warp walk one
// tile's range, so the id reads and key writes are coalesced; the depth gather is served by L2.
__global__ void __launch_bounds__(KEYS_THREADS) isect_keys_kernel(int n_tiles, const int2* __restrict__ ranges,
                                                                  const int32_t* __restrict__ ids, int64_t n_pairs,
                                                                  const float* __restrict__ depth, int64_t* __restrict__ keys) {
    const int tile = int((int64_t(blockIdx.x) * KEYS_THREADS + threadIdx.x) >> 5);
    const int lane = threadIdx.x & 31;
    if (tile >= n_tiles) return;
    const int2 r = __ldg(ranges + tile);
    const int64_t end = min(int64_t(r.y), n_pairs);
    const uint64_t hi = uint64_t(uint32_t(tile)) << 32;
    for (int64_t i = int64_t(r.x) + lane; i < end; i += 32)
        keys[i] = int64_t(hi | uint64_t(__float_as_uint(__ldg(depth + __ldg(ids + i)))));
}

// offsets[t] = index of the first key whose tile (key >> 32) is >= t: gsplat's isect_offset_encode for one camera (an empty tile
// gets the next non-empty start, tiles past the last key get n_pairs).  O(log n_pairs) reads per tile.
__global__ void __launch_bounds__(OFFSETS_THREADS) isect_offsets_kernel(int64_t n_pairs, const int64_t* __restrict__ keys, int n_tiles,
                                                                        int32_t* __restrict__ offsets) {
    const int t = blockIdx.x * OFFSETS_THREADS + threadIdx.x;
    if (t >= n_tiles) return;
    int64_t lo = 0, hi = n_pairs;
    while (lo < hi) {
        const int64_t mid = (lo + hi) >> 1;
        if ((__ldg(keys + mid) >> 32) < int64_t(t)) lo = mid + 1;
        else hi = mid;
    }
    offsets[t] = int32_t(lo);
}

}  // namespace

int launch_isect_keys(int n_tiles, const int32_t* tile_ranges, const int32_t* sorted_ids, int64_t n_pairs, const float* depth, int64_t* keys,
                      cudaStream_t s) {
    if (n_tiles == 0 || n_pairs == 0) return B200GS_OK;
    isect_keys_kernel<<<(unsigned)div_up64(int64_t(n_tiles) * 32, KEYS_THREADS), KEYS_THREADS, 0, s>>>(
        n_tiles, reinterpret_cast<const int2*>(tile_ranges), sorted_ids, n_pairs, depth, keys);
    B200GS_LAUNCH_CHECK();
    return B200GS_OK;
}

int launch_isect_offsets(int64_t n_pairs, const int64_t* keys, int n_tiles, int32_t* offsets, cudaStream_t s) {
    if (n_tiles == 0) return B200GS_OK;
    isect_offsets_kernel<<<(unsigned)div_up(n_tiles, OFFSETS_THREADS), OFFSETS_THREADS, 0, s>>>(n_pairs, keys, n_tiles, offsets);
    B200GS_LAUNCH_CHECK();
    return B200GS_OK;
}

}  // namespace b200gs
