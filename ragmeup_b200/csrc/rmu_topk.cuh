// Block-wide top-k selection over 64-bit ordered keys (rmu_ptx.cuh make_key: score descending, then row ascending;
// 0 = an empty slot): a radix select, the collection of the keys above a threshold and a bitonic sort.  Shared by
// the flat index's selection kernels and the decoder's sampler.  Include inside namespace rmu.
#pragma once

// sort s[0 .. n) descending, n a power of two.  All threads call.
__device__ __forceinline__ void block_bitonic_desc(unsigned long long* s, int n /*pow2*/) {
    for (int k = 2; k <= n; k <<= 1) {
        for (int j = k >> 1; j > 0; j >>= 1) {
            __syncthreads();
            for (int t = threadIdx.x; t < n / 2; t += blockDim.x) {
                const int i = ((t & ~(j - 1)) << 1) | (t & (j - 1));  // index with bit j clear
                const int l = i | j;
                const bool desc = ((i & k) == 0);
                unsigned long long a = s[i], b = s[l];
                const bool sw = desc ? (a < b) : (a > b);
                if (sw) { s[i] = b; s[l] = a; }
            }
        }
    }
    __syncthreads();
}

constexpr int kSel2Max = 1024;                   // keys a selection kernel collects, sorts (and re-scores), at most

// Block-wide radix select (8 bits per pass, most significant first) over passes [pass0, pass1): after pass 8 the
// state holds the ksel-th largest non-zero key among load_key(0..total); after pass 4 its 32 score bits (the low
// word still zero) and, in *s_ties, how many keys share those score bits.  *s_remaining < 0 means fewer than ksel
// keys exist ("keep everything").  pass0 == 0 initialises the state.  All threads call.
template <typename LoadKey>
__device__ __forceinline__ void block_radix_passes(LoadKey load_key, long long total, int ksel, int pass0, int pass1, int* hist,
                                                   unsigned long long* s_prefix, int* s_remaining, int* s_ties) {
    const int tid = threadIdx.x;
    if (pass0 == 0) {
        if (tid == 0) { *s_prefix = 0ull; *s_remaining = ksel; *s_ties = 0; }
        __syncthreads();
    }
    for (int pass = pass0; pass < pass1; ++pass) {
        const int shift = 56 - 8 * pass;
        for (int i = tid; i < 256; i += blockDim.x) hist[i] = 0;
        __syncthreads();
        const unsigned long long prefix = *s_prefix;
        const int remaining = *s_remaining;         // < 0: fewer than ksel keys exist, keep all
        const unsigned long long himask = pass == 0 ? 0ull : (~0ull << (shift + 8));
        if (remaining >= 0) {
            for (long long idx = tid; idx < total; idx += blockDim.x) {
                const unsigned long long key = load_key(idx);
                if (key != 0ull && (key & himask) == prefix) atomicAdd(&hist[(key >> shift) & 0xFF], 1);
            }
        }
        __syncthreads();
        if (tid == 0 && remaining >= 0) {
            int rem = remaining;
            int b = 255;
            for (; b >= 0; --b) {
                if (hist[b] >= rem) break;
                rem -= hist[b];
            }
            if (b < 0) { *s_remaining = -1; }
            else { *s_prefix = prefix | (static_cast<unsigned long long>(b) << shift); *s_remaining = rem; *s_ties = hist[b]; }
        }
        __syncthreads();
    }
}

// the ksel-th largest non-zero key, or 1 ("keep everything") when fewer than ksel exist.  Ties on the 32 score bits
// are rare: when the keys that share the selected score are all needed (s_ties == s_remaining after four passes) the
// threshold is that score with a zero row word and the four passes over the row bits are skipped.
template <typename LoadKey>
__device__ __forceinline__ unsigned long long block_radix_select(LoadKey load_key, long long total, int ksel, int* hist,
                                                                 unsigned long long* s_prefix, int* s_remaining, int* s_ties) {
    block_radix_passes(load_key, total, ksel, 0, 4, hist, s_prefix, s_remaining, s_ties);
    if (*s_remaining >= 0 && *s_ties != *s_remaining)        // uniform: shared state, read after the barrier
        block_radix_passes(load_key, total, ksel, 4, 8, hist, s_prefix, s_remaining, s_ties);
    return *s_remaining < 0 ? 1ull : *s_prefix;
}

// the non-zero keys >= T among load_key(0..total) into sel[0 .. kSel2Max), in no particular order; returns how many there
// were (more than kSel2Max were not stored).  All threads call.
template <typename LoadKey>
__device__ __forceinline__ int block_collect(LoadKey load_key, long long total, unsigned long long T, unsigned long long* sel,
                                             int* s_cnt) {
    if (threadIdx.x == 0) *s_cnt = 0;
    __syncthreads();
    for (long long idx = threadIdx.x; idx < total; idx += blockDim.x) {
        const unsigned long long key = load_key(idx);
        if (key != 0ull && key >= T) { const int pos = atomicAdd(s_cnt, 1); if (pos < kSel2Max) sel[pos] = key; }
    }
    __syncthreads();
    return *s_cnt;
}

// sort sel[0 .. n) descending (n <= kSel2Max), zero padded to a power of two >= 32.  All threads call.
__device__ __forceinline__ void block_sort_desc(unsigned long long* sel, int n) {
    int m2 = 32;
    while (m2 < n) m2 <<= 1;
    for (int i = n + threadIdx.x; i < m2; i += blockDim.x) sel[i] = 0ull;
    block_bitonic_desc(sel, m2);
}
