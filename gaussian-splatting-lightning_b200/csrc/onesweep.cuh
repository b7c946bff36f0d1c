// Hand-written device-wide primitives of the tile binning (no cub): warp and block scans, a single-pass chained scan
// (decoupled look-back on one value per block) and a stable LSD radix sort in the onesweep style — the caller builds the
// histograms of all digits in one go, then one kernel per 8-bit digit in which every tile ranks its records with warp
// ballots, publishes its digit counts, obtains its global offsets by looking back over the preceding tiles' counts, and
// scatters through a shared-memory staging area so that the global writes are runs of consecutive addresses.
//
// Records carry their key inside (a uint2 {depth key, Gaussian id} for the depth sort, a uint4 {tile mask lo, hi, id,
// coarse cell} for the partition by cell), so keys and payload move as one 8- or 16-byte vector.
// The number of records may be known only on the device (`d_n`): grids are sized for the capacity and surplus tiles exit.
#pragma once
#include "common.cuh"

namespace b200gs {
namespace sweep {

constexpr int RADIX = 256;
constexpr uint32_t FLAG_AGG = 1u << 30, FLAG_PREFIX = 2u << 30, VALUE_MASK = (1u << 30) - 1u;

__device__ __forceinline__ uint32_t ld_volatile(const uint32_t* p) {
    uint32_t v;
    asm volatile("ld.volatile.global.u32 %0, [%1];" : "=r"(v) : "l"(p));
    return v;
}
// relaxed gpu-scope load, executed only when `pred` (otherwise `dflt`): a predicated LDG, no branch around it
__device__ __forceinline__ uint32_t ld_relaxed_if(const uint32_t* p, bool pred, uint32_t dflt) {
    uint32_t v;
    asm volatile("{\n\t.reg .pred q;\n\tsetp.ne.u32 q, %2, 0;\n\tmov.u32 %0, %3;\n\t@q ld.relaxed.gpu.global.u32 %0, [%1];\n\t}"
                 : "=r"(v) : "l"(p), "r"((uint32_t)pred), "r"(dflt) : "memory");
    return v;
}
__device__ __forceinline__ void st_volatile(uint32_t* p, uint32_t v) { asm volatile("st.volatile.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory"); }

// Wait until a look-back word has been published.  Tiles take tickets in launch order, so the tile that owns the word is
// already running; the bound only turns a logic error (a word that is never published) into a trap instead of a hang.
__device__ __forceinline__ uint32_t wait_published(const uint32_t* p) {
    uint32_t v = ld_volatile(p);
    for (unsigned spins = 0; (v >> 30) == 0u; ++spins) {
        if (spins > (1u << 27)) asm volatile("trap;");
        v = ld_volatile(p);
    }
    return v;
}

__device__ __forceinline__ uint32_t key_of(const uint2& r) { return r.x; }
__device__ __forceinline__ uint32_t key_of(const uint4& r) { return r.w; }

// ---- scans -----------------------------------------------------------------------------------------------------------
// inclusive scan over the 32 lanes of a warp (all lanes call it)
template <typename T>
__device__ __forceinline__ T warp_inclusive(T v) {
    const unsigned lane = threadIdx.x & 31u;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const T t = __shfl_up_sync(0xffffffffu, v, o);
        if ((int)lane >= o) v += t;
    }
    return v;
}

// Block-wide exclusive scan of one value per thread over NW warps: returns the thread's exclusive prefix, *total = block sum
// (total may be NULL).  s_warp[NW + 1] (NW without total) is free again when it returns.  Up to 16 warps every thread sums the warp totals it needs; 32 warps scan them
// in warp 0 instead of every thread reading all 32.
template <typename T, int NW>
__device__ __forceinline__ T block_exclusive(T v, T* s_warp, T* total) {
    const unsigned lane = threadIdx.x & 31u, w = threadIdx.x >> 5;
    const T inc = warp_inclusive(v);
    if (lane == 31) s_warp[w] = inc;
    __syncthreads();
    T base = 0, tot = 0;
    if (NW <= 16) {
#pragma unroll
        for (int k = 0; k < NW; ++k) {
            const T c = s_warp[k];
            base += (k < (int)w) ? c : T(0);
            tot += c;
        }
    } else {
        static_assert(NW <= 32, "one warp scans the warp totals");
        if (w == 0) {
            const T c = (int)lane < NW ? s_warp[lane] : T(0);
            const T winc = warp_inclusive(c);
            s_warp[lane] = winc - c;
            if (total != nullptr && lane == 31) s_warp[NW] = winc;     // the slot costs chunk_prefix_kernel 2 registers
        }
        __syncthreads();
        base = s_warp[w];
        if (total != nullptr) tot = s_warp[NW];
    }
    const T excl = base + inc - v;
    __syncthreads();
    if (total != nullptr) *total = tot;
    return excl;
}

// Exclusive prefix of one 30-bit value per tile over the tiles in ticket order.  `state[t]` must be zero before the launch.
// Called by ALL 32 lanes of ONE warp (same arguments); returns (to every lane) the sum of the values of tiles 0..t-1.
// The look-back is warp-wide: lane l loads tiles p - l - 32 j, j < depth, all loads in flight together; the walk stops at the
// nearest tile that has already published its inclusive prefix and resumes at the first word that is not published yet.
// depth ramps 1 -> 2 -> 4 words per lane (32 -> 64 -> 128 predecessors per step) while every word read is published: in the
// steady state of a long grid the nearest predecessor's prefix is out already and wide steps only waste L2 requests, while a
// whole wave of tiles that starts at once has no prefix yet and tile t needs about t / 128 round trips to L2.
__device__ __forceinline__ uint32_t chained_exclusive(uint32_t* state, int t, uint32_t value) {
    constexpr int DEPTH = 4;
    const unsigned lane = threadIdx.x & 31u;
    if (lane == 0) st_volatile(state + t, (value & VALUE_MASK) | (t == 0 ? FLAG_PREFIX : FLAG_AGG));
    uint32_t acc = 0;                 // per-lane partial sum, reduced once at the end
    bool done = (t == 0);
    unsigned spins = 0;
    int depth = 1;
    for (int p = t - 1; !done;) {
        uint32_t v[DEPTH];
#pragma unroll
        for (int j = 0; j < DEPTH; ++j) {
            const int idx = p - (int)lane - 32 * j;
            v[j] = (j >= depth) ? 0u : (idx >= 0 ? ld_volatile(state + idx) : FLAG_PREFIX);      // before tile 0: an empty prefix
        }
        int consumed = 0;
        bool stalled = false;
#pragma unroll
        for (int j = 0; j < DEPTH; ++j) {
            if (!done && !stalled && j < depth) {
                const unsigned pub = __ballot_sync(0xffffffffu, (v[j] >> 30) != 0u);
                const unsigned pre = __ballot_sync(0xffffffffu, (v[j] & FLAG_PREFIX) != 0u);
                const int n_pub = (pub == 0xffffffffu) ? 32 : __ffs(~pub) - 1;     // run of published words, nearest first
                const int first_pre = pre ? __ffs(pre) - 1 : 32;
                const int take = min(n_pub, first_pre + 1);
                acc += ((int)lane < take) ? (v[j] & VALUE_MASK) : 0u;
                consumed += take;
                done = first_pre < n_pub;
                stalled = !done && n_pub < 32;
            }
        }
        p -= consumed;
        if (!stalled) depth = min(2 * depth, DEPTH);
        if (consumed == 0 && ++spins > (1u << 27)) asm volatile("trap;");   // a word that is never published: a logic error, not a hang
    }
    acc = warp_reduce<Sum>(acc);
    if (lane == 0 && t > 0) st_volatile(state + t, ((acc + value) & VALUE_MASK) | FLAG_PREFIX);
    return acc;
}

// The block's ticket: blocks are numbered in the order they start, so every block a chained scan waits for is already running.
__device__ __forceinline__ int block_ticket(uint32_t* ticket) {
    __shared__ int s_tile;
    if (threadIdx.x == 0) s_tile = (int)atomicAdd(ticket, 1u);
    __syncthreads();
    return s_tile;
}

// Device-wide exclusive scan of one int per thread over the blocks in ticket order t (NW warps per block): block scan, chained
// scan of the block totals, returns the thread's global exclusive prefix.
template <int NW>
__device__ __forceinline__ uint32_t chained_block_exclusive(int v, uint32_t* state, int t) {
    __shared__ int s_warp[NW + 1];
    __shared__ uint32_t s_excl;
    int block_total;
    const int local = block_exclusive<int, NW>(v, s_warp, &block_total);
    if (threadIdx.x < 32) {
        const uint32_t excl = chained_exclusive(state, t, (uint32_t)block_total);
        if (threadIdx.x == 0) s_excl = excl;
    }
    __syncthreads();
    return s_excl + (uint32_t)local;
}

// ---- one digit pass ----------------------------------------------------------------------------------------------------
// hist[RADIX]: global count of every digit value of this pass; lookback[tiles][RADIX] and *ticket zero before the launch.
// PASS_THREADS threads per tile, IPT records per thread (tile = 4096 8-byte or 2048 16-byte records: 32 KB of staging).  16 warps
// per tile and <= 64 registers keep two tiles = 32 warps resident per SM: the ranking loop is a chain of dependent shared-memory
// read-modify-writes per warp, latency that only other warps can hide (256 threads x 16 records at 127 registers left most issue
// slots idle).
constexpr int PASS_THREADS = 512;
constexpr int PASS_WARPS = PASS_THREADS / 32;

template <typename Rec, int IPT>
__global__ void __launch_bounds__(PASS_THREADS, 2) onesweep_pass_kernel(const Rec* __restrict__ in, Rec* __restrict__ out, const int64_t* __restrict__ d_n,
                                                                        int64_t cap, int shift, const uint32_t* __restrict__ hist,
                                                                        uint32_t* __restrict__ lookback, uint32_t* __restrict__ ticket) {
    constexpr int TILE_ITEMS = PASS_THREADS * IPT;
    static_assert(TILE_ITEMS < 65536, "per-warp digit counts are 16-bit");
    __shared__ unsigned short s_cnt[PASS_WARPS][RADIX];   // per-warp digit counts -> offsets of the warp inside the tile's digit run
    __shared__ int s_base[RADIX];                         // global index of the tile's first record of a digit, minus its slot in the tile
    __shared__ int s_scan[PASS_WARPS + 1];
    __shared__ int s_tile;
    __shared__ Rec s_stage[TILE_ITEMS];
    const int64_t n = d_n ? min(cap, *d_n) : cap;
    const int tid = threadIdx.x;
    const unsigned lane = tid & 31u, w = tid >> 5;
    if (tid == 0) s_tile = (int)atomicAdd(ticket, 1u);
    for (int i = tid; i < PASS_WARPS * RADIX / 2; i += PASS_THREADS) reinterpret_cast<uint32_t*>(&s_cnt[0][0])[i] = 0;
    __syncthreads();
    const int t = s_tile;
    const int64_t tile_lo = int64_t(t) * TILE_ITEMS;
    if (tile_lo >= n) return;
    const int tile_n = (int)min((int64_t)TILE_ITEMS, n - tile_lo);

    Rec rec[IPT];
    int dig[IPT];      // 0..255, or 256 for the slots past the end
    int rank[IPT];
    unsigned short* my_cnt = s_cnt[w];
#pragma unroll
    for (int i = 0; i < IPT; ++i) {
        const int local = (int)w * (32 * IPT) + i * 32 + (int)lane;
        const bool valid = local < tile_n;
        if (valid) rec[i] = in[tile_lo + local];
        dig[i] = valid ? (int)((key_of(rec[i]) >> shift) & 255u) : 256;
    }
    // Lanes with the same digit.  `match.any` peels one distinct value per round: with ~30 distinct 8-bit digits in a warp ranking
    // took most of a tile's time.  Eight ballots
    // (one per digit bit, plus one for the slots past the end) cost the same whatever the digits are, and the ballots of the IPT
    // records are independent of each other: they pipeline, only the counter updates below are a dependent chain.
    unsigned peers[IPT];
#pragma unroll
    for (int i = 0; i < IPT; ++i) {
        const bool valid = dig[i] < 256;
        const unsigned mv = __ballot_sync(0xffffffffu, valid);
        unsigned pm = valid ? mv : ~mv;
#pragma unroll
        for (int b = 0; b < 8; ++b) {
            const bool bit = (dig[i] >> b) & 1;
            const unsigned m = __ballot_sync(0xffffffffu, bit);
            pm &= bit ? m : ~m;
        }
        peers[i] = pm;
    }
#pragma unroll
    for (int i = 0; i < IPT; ++i) {
        const int lt = __popc(peers[i] & ((1u << lane) - 1u));
        int before = 0;
        if (dig[i] < 256) before = my_cnt[dig[i]];
        __syncwarp();
        if (dig[i] < 256 && lt == 0) my_cnt[dig[i]] = (unsigned short)(before + __popc(peers[i]));
        __syncwarp();
        rank[i] = before + lt;
    }
    __syncthreads();
    // thread d (< RADIX) owns digit d: offsets of the warps inside the digit's run, the tile's count
    uint32_t run = 0;
    uint32_t* col = lookback + (tid & (RADIX - 1));                        // lookback[p * RADIX + d]
    if (tid < RADIX) {
#pragma unroll
        for (int k = 0; k < PASS_WARPS; ++k) {
            const uint32_t c = s_cnt[k][tid];
            s_cnt[k][tid] = (unsigned short)run;
            run += c;
        }
        st_volatile(col + int64_t(t) * RADIX, (run & VALUE_MASK) | (t == 0 ? FLAG_PREFIX : FLAG_AGG));
    }
    int tot;
    const int tile_start = block_exclusive<int, PASS_WARPS>((int)run, s_scan, &tot);                              // first slot of digit d in the staged tile
    if (tid < RADIX) {
        // slot of a record = tile_start[d] + warp offset + rank; fold tile_start into the warp offsets
#pragma unroll
        for (int k = 0; k < PASS_WARPS; ++k) s_cnt[k][tid] = (unsigned short)(s_cnt[k][tid] + tile_start);
    }
    __syncthreads();
    // the records go to their slot of the staged tile BEFORE the look-back: the slot does not depend on the other tiles, and the
    // look-back then has the registers of the records for its loads
#pragma unroll
    for (int i = 0; i < IPT; ++i)
        if (dig[i] < 256) s_stage[my_cnt[dig[i]] + rank[i]] = rec[i];
    // look-back over the preceding tiles' words of digit d: LB predicated relaxed loads in flight per step (before tile 0 a word
    // reads as an empty prefix).  The run of published words up to the nearest prefix is summed; a word that is not published yet
    // ends the step and the walk resumes there.  On a pass over 0.65 M / 2.3 M 8-byte records a fixed 8 per step beat both batches
    // doubling from 4 to 32 and a fixed 32: the wide batches cost more in L2 requests than they save in round trips.
    constexpr int LB = 8;
    uint32_t before_tiles = 0;
    if (tid < RADIX) {
        for (int p = t - 1; p >= 0;) {
            uint32_t v[LB];
#pragma unroll
            for (int k = 0; k < LB; ++k) v[k] = ld_relaxed_if(col + int64_t(max(p - k, 0)) * RADIX, p - k >= 0, FLAG_PREFIX);
            int used = 0;
            bool done = false, open = true;
#pragma unroll
            for (int k = 0; k < LB; ++k) {
                const bool pub = (v[k] >> 30) != 0u;
                open = open && !done && pub;                               // still inside the run of published words, before any prefix
                before_tiles += open ? (v[k] & VALUE_MASK) : 0u;
                used += open ? 1 : 0;
                done = done || (open && (v[k] & FLAG_PREFIX) != 0u);
            }
            if (done) break;
            p -= used;
            if (used == 0 && p >= 0) {     // the nearest word is not out yet: wait for it, then go on from the next one
                const uint32_t w0 = wait_published(col + int64_t(p) * RADIX);
                before_tiles += w0 & VALUE_MASK;
                if (w0 & FLAG_PREFIX) break;
                --p;
            }
        }
        if (t > 0) st_volatile(col + int64_t(t) * RADIX, ((before_tiles + run) & VALUE_MASK) | FLAG_PREFIX);
    }
    const int digit_start = block_exclusive<int, PASS_WARPS>(tid < RADIX ? (int)hist[tid] : 0, s_scan, &tot);   // first global index of digit d
    if (tid < RADIX) s_base[tid] = digit_start + (int)before_tiles - tile_start;
    __syncthreads();
    for (int s = tid; s < tile_n; s += PASS_THREADS) {
        const Rec r = s_stage[s];
        const int d = (int)((key_of(r) >> shift) & 255u);
        out[s_base[d] + s] = r;
    }
}

}  // namespace sweep
}  // namespace b200gs
