// xmr_ragged.cuh -- ragged batches of SHA-256, CRC16 and quicksort (COAST_UNIT_OFFSETS in coast_rt.h).
//
// n messages lie end to end in one buffer; n + 1 u64 byte offsets say where each starts.  Unit u hashes d_in[off[u] ..
// off[u+1]) with exactly what a single-unit launch of that length does (same compressions / byte steps, same fault sites,
// same votes and counters), so the per-message bodies reuse the building blocks of xmr_sha256.cuh and xmr_crc16.cuh.
// Quicksort units are int32 arrays, sorted into the same byte range of d_out by the state machine of xmr_qsort.cuh.
//
// Schedule.  A warp runs as long as its longest unit, so with mixed lengths the lanes of short units idle.  A stream-ordered
// counting sort orders the units by cost first (xmr_ragged_hist -> xmr_ragged_scan -> xmr_ragged_scatter: a histogram with
// shared-memory atomics, a one-CTA exclusive scan in DESCENDING cost order, a scatter into a u32 permutation).  The unit
// kernels then run a persistent grid whose warps pull warp-tiles of consecutive permuted units from a counter: neighbours
// in a tile cost about the same, the longest units go first and the short ones fill the tail.  The order inside a bucket may
// differ between runs; nothing observable depends on it (every unit is independent, first_fault_unit is a minimum).
//
// Loads.  Messages start at any byte offset.  Words are assembled from aligned 4-byte loads (byte_perm across two words),
// and a word is only loaded when it holds a byte of the message.
#pragma once
#include "xmr_sha256.cuh"
#include "xmr_crc16.cuh"
#include "xmr_qsort.cuh"

namespace xmr {

struct RaggedHdr {
    const unsigned long long* off;   // the caller's offset table (written by xmr_ragged_scan)
    unsigned int next;               // next warp-tile to hand out
};
static_assert(sizeof(RaggedHdr) <= XMR_RAGGED_HDR && XMR_RAGGED_SCAN_THREADS == XMR_RAGGED_BUCKETS,
              "the header fits its slot; the scan has one thread per cost bucket");

// Offset u as a unit boundary.  Units of ELEM-byte elements (quicksort: 4) start on element boundaries: the low bits of an
// offset are ignored, so a malformed table never makes a unit load or store a misaligned element.
template <uint32_t ELEM = 1u>
__device__ __forceinline__ unsigned long long ragged_at(const unsigned long long* off, unsigned long long u) {
    return __ldg(off + u) & ~(unsigned long long)(ELEM - 1u);
}
// length of unit u in bytes, clamped to [0, bound]; a decreasing pair counts as 0, so a malformed table never makes a unit read
// past off[u] + bound.  The pre-pass and the kernels both take it from here, so the sort key and a unit's length agree.
template <uint32_t ELEM = 1u>
__device__ __forceinline__ uint32_t ragged_len(const unsigned long long* off, unsigned long long u, uint32_t bound) {
    const unsigned long long o0 = ragged_at<ELEM>(off, u), o1 = ragged_at<ELEM>(off, u + 1);
    return o1 > o0 ? (o1 - o0 < bound ? (uint32_t)(o1 - o0) : bound) : 0u;
}
// sort key of a unit of len bytes (XMR_RAGGED_COST_*): bytes for CRC16, compressions for SHA-256 and elements for quicksort
// (the top bucket takes everything longer)
__device__ __forceinline__ uint32_t ragged_cost(uint32_t len, uint32_t kind) {
    if (kind == XMR_RAGGED_COST_CRC) return len;
    const uint32_t c = kind == XMR_RAGGED_COST_SHA ? (len + 8u) / 64u + 1u : len / 4u;
    return c < XMR_RAGGED_BUCKETS - 1u ? c : XMR_RAGGED_BUCKETS - 1u;
}
__device__ __forceinline__ uint32_t ragged_unit_cost(const unsigned long long* off, unsigned long long u, uint32_t bound, uint32_t kind) {
    return ragged_cost(kind == XMR_RAGGED_COST_QSORT ? ragged_len<4>(off, u, bound) : ragged_len(off, u, bound), kind);
}

// The next warp-tile of this warp (uniform), from the counter in the scratch header.
__device__ __forceinline__ uint32_t ragged_pull(RaggedHdr* hdr, int lane) {
    uint32_t wt = 0;
    if (lane == 0) wt = atomicAdd(&hdr->next, 1u);
    return __shfl_sync(0xFFFFFFFFu, wt, 0);
}

// store_vote_bytes for a per-lane byte count: every lane shuffles whatever its nb (units of one warp differ in length); the
// value is only replaced where there are bytes to vote
template <int NC>
__device__ __forceinline__ uint32_t ragged_vote_bytes(uint32_t& x, uint32_t nb, int lane, bool majority) {
    if (NC == 1) return 0u;
    const uint32_t live = nb ? 0xFFFFFFFFu << (8u * (4u - nb)) : 0u;
    const int base = Lanes<NC>::unit(lane) * NC;
    const uint32_t r0 = __shfl_sync(0xFFFFFFFFu, x, base), r1 = __shfl_sync(0xFFFFFFFFu, x, base + 1);
    const uint32_t e01 = __vcmpeq4(r0, r1);
    if (NC == 2) return __popc(~e01 & live) >> 3;
    const uint32_t r2 = __shfl_sync(0xFFFFFFFFu, x, base + 2);
    const uint32_t e02 = __vcmpeq4(r0, r2);
    if (nb) x = majority ? ((r0 & r1) | (r0 & r2) | (r1 & r2)) : ((r0 & e01) | (r2 & ~e01));
    return __popc(~(e01 & e02) & live) >> 3;
}

// Block `blk` of a len-byte message at `msg` (any alignment) as the big-endian words sha256_transform packs (:34-40), with
// the 0x80 byte and the 64-bit bit count of the padding (:132-163) in place.
__device__ __forceinline__ void sha_var_block(uint32_t (&m)[16], const uint8_t* msg, uint32_t len, uint32_t blk, uint32_t nblk) {
    const uint32_t p = blk * 64u;
    const uintptr_t a = reinterpret_cast<uintptr_t>(msg) + p, end = reinterpret_cast<uintptr_t>(msg) + len;
    const uint32_t s = (uint32_t)a & 3u, sel = 0x3210u + 0x1111u * s;
    const uint32_t* w = reinterpret_cast<const uint32_t*>(a - s);
    uint32_t lo = a < end ? __ldg(w) : 0u;                    // holds byte a
#pragma unroll
    for (int i = 0; i < 16; ++i) {
        const uint32_t hi = reinterpret_cast<uintptr_t>(w + i + 1) < end ? __ldg(w + i + 1) : 0u;
        uint32_t v = __byte_perm(lo, hi, sel);                // little-endian bytes p + 4i .. p + 4i + 3
        lo = hi;
        const int k = (int)len - (int)(p + 4u * i);           // message bytes in this word (len <= 2^28)
        if (k < 4) v = k <= 0 ? (k == 0 ? 0x80u : 0u) : ((v & ((1u << (8 * k)) - 1u)) | (0x80u << (8 * k)));
        m[i] = bswap(v);
    }
    if (blk == nblk - 1u) { m[14] = len >> 29; m[15] = len << 3; }   // :155-163
}

template <int NC, bool INJECT>
__device__ __forceinline__ void sha256_var_body(const xmr_args& a) {
    constexpr int UPW = Lanes<NC>::kUnitsPerWarp;
    const int lane = threadIdx.x & 31;
    const int r = Lanes<NC>::replica(lane);
    RaggedHdr* hdr = reinterpret_cast<RaggedHdr*>(const_cast<void*>(a.aux));
    const unsigned long long* off = hdr->off;
    const uint32_t* perm = reinterpret_cast<const uint32_t*>(static_cast<const uint8_t*>(a.aux) + XMR_RAGGED_PERM);
    const uint8_t* in = static_cast<const uint8_t*>(a.in);
    const unsigned long long n_wtiles = (a.n_units + UPW - 1) / UPW;
    const bool sv = (a.flags & XMR_F_STORE_VOTES) != 0;
    const bool majority = a.flags & COAST_F_MAJORITY_VOTER;
    Tally tally(a);
    for (uint32_t wt = ragged_pull(hdr, lane); wt < n_wtiles; wt = ragged_pull(hdr, lane)) {
        const unsigned long long pos = (unsigned long long)wt * UPW + Lanes<NC>::unit(lane);
        const bool valid = pos < a.n_units;
        const unsigned long long local = valid ? __ldg(perm + pos) : 0ull;
        const uint32_t len = valid ? ragged_len(off, local, a.unit_bytes) : 0u;
        const uint8_t* msg = in + __ldg(off + local);
        const uint32_t nblk = (len + 8u) / 64u + 1u;
        const unsigned long long gunit = a.unit_base + local;
        uint32_t fsite = 0xFFFFFFFFu, fmask = 0u;
        if (INJECT) {
            Fault f = fault_for_unit(a, NC, local, SHA_SITES_PER_BLOCK * nblk, [](uint32_t) { return 32u; });
            if (f.active && valid) {
                if (Lanes<NC>::voter(lane)) tally.injected++;
                if ((int)f.replica == r) { fmask = 1u << f.bit; fsite = f.site; }
            }
        }
        uint32_t st[8];
        sha_init(st);
        if (!sv) {
            for (uint32_t blk = 0; blk < nblk; ++blk) {       // lanes diverge here and meet again at the vote
                uint32_t m[16];
                sha_var_block(m, msg, len, blk, nblk);
                const uint32_t fs = (INJECT && fsite / SHA_SITES_PER_BLOCK == blk) ? fsite % SHA_SITES_PER_BLOCK : 0xFFFFFFFFu;
                sha_compress<INJECT>(st, m, fs, fmask);
            }
            sha_vote_store<NC>(st, static_cast<uint8_t*>(a.out), local, gunit, valid, lane, a.flags, tally);
        } else {
            // in-loop store votes shuffle across the warp: every lane walks the warp's longest unit and keeps only its own
            // blocks (a unit's replicas always agree on whether a block is theirs)
            const uint32_t wblk = __reduce_max_sync(0xFFFFFFFFu, nblk);
            uint32_t sv_bad = 0;
            for (uint32_t blk = 0; blk < wblk; ++blk) {
                const bool act = blk < nblk;
                uint32_t m[16];
                if (act) sha_var_block(m, msg, len, blk, nblk);
                else {
#pragma unroll
                    for (int i = 0; i < 16; ++i) m[i] = 0u;
                }
                const uint32_t lo = blk * 64u, nmsg = len > lo ? (len - lo < 64u ? len - lo : 64u) : 0u;
                uint32_t bad = 0;
#pragma unroll
                for (int w = 0; w < 16; ++w) {                // ctx_data[k] = data[i] (:120), one u8 vote per message byte
                    const uint32_t nb = nmsg > 4u * w ? (nmsg - 4u * w < 4u ? nmsg - 4u * w : 4u) : 0u;
                    bad += ragged_vote_bytes<NC>(m[w], nb, lane, majority);
                }
                const uint32_t fs = (INJECT && fsite / SHA_SITES_PER_BLOCK == blk) ? fsite % SHA_SITES_PER_BLOCK : 0xFFFFFFFFu;
                uint32_t keep[8];
#pragma unroll
                for (int i = 0; i < 8; ++i) keep[i] = st[i];
                bad += sha_compress_sv<NC, INJECT>(st, m, fs, fmask, lane, majority);
                if (act) sv_bad += bad;
                else {
#pragma unroll
                    for (int i = 0; i < 8; ++i) st[i] = keep[i];
                }
            }
            uint32_t o[8], bad = 0;                           // the SoR exit: len + 720 per compression + 32 votes
#pragma unroll
            for (int i = 0; i < 8; ++i) { Voted v = vote_u32<NC, 1>(st[i], majority); o[i] = bswap(v.vote); bad += v.bad; }
            if (valid && Lanes<NC>::voter(lane)) {
                uint4* dst = reinterpret_cast<uint4*>(static_cast<uint8_t*>(a.out) + local * 32ull);
                dst[0] = make_uint4(o[0], o[1], o[2], o[3]);
                dst[1] = make_uint4(o[4], o[5], o[6], o[7]);
                tally.unit_exit<NC>(bad + sv_bad, len + 720u * nblk + 32u, a.flags, gunit);
            }
        }
    }
    tally.flush(a.counters);
}

// CRC16 of a ragged batch: the general path's table form of the byte step (T replicated over the lanes in shared memory),
// bytes taken out of aligned words.
template <int NC, bool INJECT>
__device__ __forceinline__ void crc16_var_body(const xmr_args& a) {
    constexpr int UPW = Lanes<NC>::kUnitsPerWarp;
    __shared__ uint32_t tab[256 * 32];
    for (int i = threadIdx.x; i < 256 * 32; i += blockDim.x) tab[i] = crc16_step(0u, (uint32_t)i >> 5);
    __syncthreads();
    const int lane = threadIdx.x & 31;
    const uint32_t* const tl = tab + lane;
    const int r = Lanes<NC>::replica(lane);
    RaggedHdr* hdr = reinterpret_cast<RaggedHdr*>(const_cast<void*>(a.aux));
    const unsigned long long* off = hdr->off;
    const uint32_t* perm = reinterpret_cast<const uint32_t*>(static_cast<const uint8_t*>(a.aux) + XMR_RAGGED_PERM);
    const uint8_t* in = static_cast<const uint8_t*>(a.in);
    const unsigned long long n_wtiles = (a.n_units + UPW - 1) / UPW;
    Tally tally(a);
    for (uint32_t wt = ragged_pull(hdr, lane); wt < n_wtiles; wt = ragged_pull(hdr, lane)) {
        const unsigned long long pos = (unsigned long long)wt * UPW + Lanes<NC>::unit(lane);
        const bool valid = pos < a.n_units;
        const unsigned long long local = valid ? __ldg(perm + pos) : 0ull;
        const uint32_t len = valid ? ragged_len(off, local, a.unit_bytes) : 0u;
        const uintptr_t msg = reinterpret_cast<uintptr_t>(in + __ldg(off + local));
        const unsigned long long gunit = a.unit_base + local;
        uint32_t fsite = 0xFFFFFFFFu, fmask = 0u;
        if (INJECT) {
            Fault f = fault_for_unit(a, NC, local, 2u * len, CrcWidth{len});
            if (f.active && valid) {
                if (Lanes<NC>::voter(lane)) tally.injected++;
                if ((int)f.replica == r) { fsite = f.site; fmask = 1u << f.bit; }
            }
        }
        uint32_t crc = 0xFFFFu, w = 0;
        if (!(a.flags & XMR_F_STORE_VOTES)) {
            for (uint32_t i = 0; i < len; ++i) {
                const uintptr_t p = msg + i;
                if (i == 0 || (p & 3u) == 0) w = __ldg(reinterpret_cast<const uint32_t*>(p & ~(uintptr_t)3));
                uint32_t b = (w >> (8u * (uint32_t)(p & 3u))) & 0xFFu;
                if (INJECT && fsite == len + i) b ^= fmask;
                crc = ((crc << 8) & 0xFFFFu) ^ tl[(((crc >> 8) ^ b) & 0xFFu) << 5];
                if (INJECT && fsite == i) crc ^= fmask;
            }
            crc_vote_store<NC>(crc, static_cast<uint16_t*>(a.out), local, gunit, valid, lane, a.flags, tally);
        } else {
            // the three voted assignments of crc16.c:26-28 and the SoR exit, every lane walking the warp's longest unit
            const bool majority = a.flags & COAST_F_MAJORITY_VOTER;
            const uint32_t wlen = __reduce_max_sync(0xFFFFFFFFu, len);
            uint32_t bad = 0;
            for (uint32_t i = 0; i < wlen; ++i) {
                const bool act = i < len;
                uint32_t b = 0;
                if (act) {
                    const uintptr_t p = msg + i;
                    if (i == 0 || (p & 3u) == 0) w = __ldg(reinterpret_cast<const uint32_t*>(p & ~(uintptr_t)3));
                    b = (w >> (8u * (uint32_t)(p & 3u))) & 0xFFu;
                }
                if (INJECT && fsite == len + i) b ^= fmask;
                uint32_t x = ((crc >> 8) ^ b) & 0xFFu;                                  // :26
                uint32_t bb = store_vote<NC>(x, lane, majority);
                x = (x ^ (x >> 4)) & 0xFFu;                                             // :27
                bb += store_vote<NC>(x, lane, majority);
                uint32_t c = ((crc << 8) ^ (x << 12) ^ (x << 5) ^ x) & 0xFFFFu;         // :28
                bb += store_vote<NC>(c, lane, majority);
                if (act) {
                    crc = c; bad += bb;
                    if (INJECT && fsite == i) crc ^= fmask;
                }
            }
            bad += store_vote<NC>(crc, lane, majority);                                 // :30
            if (valid && Lanes<NC>::voter(lane)) {
                static_cast<uint16_t*>(a.out)[local] = (uint16_t)crc;
                tally.unit_exit<NC>(bad, 3u * len + 1u, a.flags, gunit);
            }
        }
    }
    tally.flush(a.counters);
}

// Quicksort of a ragged batch: the state machine of xmr_qsort.cuh (qsort_step, qsort_exit) over cost-ordered warp-tiles.
// Unit u sorts the int32 elements d_in[off[u] .. off[u+1]) (offsets rounded down to a multiple of 4) into the same bytes of
// d_out.  Each lane group keeps its NC x L copies in a slot of NC x bound elements (scratch from xmr_ragged_slots); a zero-length
// unit executes its one `if (len < 2) return;` and stores nothing.
template <int NC, bool INJECT>
__device__ __forceinline__ void qsort_var_body(const xmr_args& a) {
    constexpr int UPW = Lanes<NC>::kUnitsPerWarp;
    const int lane = threadIdx.x & 31;
    const bool spare = NC == 3 && lane >= 30;                   // the two idle TMR lanes only take part in the ballots
    const int u = spare ? 0 : lane / NC, r = spare ? 0 : lane % NC, base = u * NC;
    const uint32_t gmask = spare ? 0u : (((1u << NC) - 1u) << base);
    const unsigned long long gwarp = ((unsigned long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    RaggedHdr* hdr = reinterpret_cast<RaggedHdr*>(const_cast<void*>(a.aux));
    const unsigned long long* off = hdr->off;
    const uint32_t* perm = reinterpret_cast<const uint32_t*>(static_cast<const uint8_t*>(a.aux) + XMR_RAGGED_PERM);
    const unsigned long long n_wtiles = (a.n_units + UPW - 1) / UPW;
    const uint32_t Lb = a.unit_bytes >> 2;                      // the bound in elements
    const bool majority = (a.flags & COAST_F_MAJORITY_VOTER) != 0;
    Tally tally(a);
    int32_t* const Au = reinterpret_cast<int32_t*>(static_cast<uint8_t*>(const_cast<void*>(a.aux)) + xmr_ragged_slots(a.n_units)) +
                        (gwarp * 32ull + (unsigned)base) * Lb;  // this lane group's NC x Lb slot
    auto at = [&](uint32_t e) -> int32_t& { return Au[e * NC + (uint32_t)r]; };                  // element e of this replica
    uint32_t stack[QS_MAX];                                     // (off << 16) | len, len <= 1024 needs 11 bits
    for (uint32_t wt = ragged_pull(hdr, lane); wt < n_wtiles; wt = ragged_pull(hdr, lane)) {
        const unsigned long long pos = (unsigned long long)wt * UPW + u;
        const bool valid = !spare && pos < a.n_units;
        const unsigned long long local = valid ? __ldg(perm + pos) : 0ull;
        const uint32_t L = valid ? ragged_len<4>(off, local, a.unit_bytes) / 4u : 0u;
        const unsigned long long o = valid ? ragged_at<4>(off, local) : 0ull;
        uint32_t fsite = 0xFFFFFFFFu, fmask = 0u;
        if (valid) {
            const int32_t* src = reinterpret_cast<const int32_t*>(static_cast<const uint8_t*>(a.in) + o);
            for (uint32_t e = 0; e < L; ++e) at(e) = __ldg(src + e);
            if (INJECT) {
                Fault f = fault_for_unit(a, NC, local, 33u * L, [](uint32_t) { return 32u; });
                if (f.active) {
                    if (r == 0) tally.injected++;
                    if ((int)f.replica == r) { fsite = f.site; fmask = 1u << f.bit; }
                }
                if (fsite >= 32u * L && fsite != 0xFFFFFFFFu) at(fsite - 32u * L) ^= (int32_t)fmask;
            }
        }
        QsState s;
        s.phase = valid ? QS_POP : QS_DONE;
        if (valid) stack[s.sp++] = L;                           // quick_sort(A, n): off = 0
        __syncwarp();
        while (__any_sync(0xFFFFFFFFu, s.phase != QS_DONE)) qsort_step<NC, INJECT>(s, at, stack, base, majority, fsite, fmask);
        if (valid)
            qsort_exit<NC>(a, tally, s, at, L, reinterpret_cast<int32_t*>(static_cast<uint8_t*>(a.out) + o), local, gmask, base, r, majority);
        __syncwarp();
    }
    tally.flush(a.counters);
}

}  // namespace xmr

// ---- the cost-ordering pre-pass (scratch layout in xmr_geom.h); `kind` is an XMR_RAGGED_COST_* ----
extern "C" __global__ void __launch_bounds__(XMR_CTA_THREADS)
xmr_ragged_hist(const unsigned long long* off, unsigned long long n, unsigned int bound, unsigned int kind, unsigned char* scratch) {
    __shared__ unsigned int h[XMR_RAGGED_BUCKETS];
    for (unsigned i = threadIdx.x; i < XMR_RAGGED_BUCKETS; i += blockDim.x) h[i] = 0u;
    __syncthreads();
    const unsigned long long stride = (unsigned long long)gridDim.x * blockDim.x;
    for (unsigned long long u = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; u < n; u += stride)
        atomicAdd(&h[xmr::ragged_unit_cost(off, u, bound, kind)], 1u);
    __syncthreads();
    unsigned int* cnt = reinterpret_cast<unsigned int*>(scratch + XMR_RAGGED_HDR);
    for (unsigned i = threadIdx.x; i < XMR_RAGGED_BUCKETS; i += blockDim.x)
        if (h[i]) atomicAdd(cnt + i, h[i]);
}

// bucket counts -> each bucket's first slot, buckets in descending cost order; the header gets the table and a zero counter
extern "C" __global__ void __launch_bounds__(XMR_RAGGED_SCAN_THREADS)
xmr_ragged_scan(const unsigned long long* off, unsigned char* scratch) {
    __shared__ unsigned int warp_sum[XMR_RAGGED_SCAN_THREADS / 32];
    unsigned int* cnt = reinterpret_cast<unsigned int*>(scratch + XMR_RAGGED_HDR);
    const int t = threadIdx.x, lane = t & 31, w = t >> 5;
    const int b = (int)XMR_RAGGED_BUCKETS - 1 - t;
    const unsigned int c = cnt[b];
    unsigned int x = c;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) { const unsigned int y = __shfl_up_sync(0xFFFFFFFFu, x, d); if (lane >= d) x += y; }
    if (lane == 31) warp_sum[w] = x;
    __syncthreads();
    if (w == 0) {
        unsigned int s = warp_sum[lane];
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) { const unsigned int y = __shfl_up_sync(0xFFFFFFFFu, s, d); if (lane >= d) s += y; }
        warp_sum[lane] = s;
    }
    __syncthreads();
    cnt[b] = (w ? warp_sum[w - 1] : 0u) + x - c;
    if (t == 0) {
        xmr::RaggedHdr* hdr = reinterpret_cast<xmr::RaggedHdr*>(scratch);
        hdr->off = off;
        hdr->next = 0u;
    }
}

// units -> permutation slots; one atomic per bucket present in a warp (lanes with equal cost share it)
extern "C" __global__ void __launch_bounds__(XMR_CTA_THREADS)
xmr_ragged_scatter(const unsigned long long* off, unsigned long long n, unsigned int bound, unsigned int kind, unsigned char* scratch) {
    unsigned int* next = reinterpret_cast<unsigned int*>(scratch + XMR_RAGGED_HDR);
    unsigned int* perm = reinterpret_cast<unsigned int*>(scratch + XMR_RAGGED_PERM);
    const int lane = threadIdx.x & 31;
    const unsigned long long stride = (unsigned long long)gridDim.x * blockDim.x;
    for (unsigned long long base = (unsigned long long)blockIdx.x * blockDim.x + (threadIdx.x & ~31u); base < n; base += stride) {
        const unsigned long long u = base + lane;
        const bool act = u < n;
        const unsigned int live = __ballot_sync(0xFFFFFFFFu, act);
        if (act) {
            const unsigned int b = xmr::ragged_unit_cost(off, u, bound, kind);
            const unsigned int peers = __match_any_sync(live, b);
            const int leader = __ffs(peers) - 1;
            unsigned int slot = 0u;
            if (lane == leader) slot = atomicAdd(next + b, (unsigned int)__popc(peers));
            slot = __shfl_sync(peers, slot, leader);
            perm[slot + __popc(peers & ((1u << lane) - 1u))] = (unsigned int)u;
        }
    }
}

#define XMR_SHA_VAR_KERNEL(NC, INJ)                                                                      \
    extern "C" __global__ void __launch_bounds__(XMR_CTA_THREADS)                                        \
    xmr_sha256_var_inj##INJ##_nc##NC(const __grid_constant__ xmr_args a) {                               \
        xmr::sha256_var_body<NC, INJ != 0>(a);                                                           \
    }
#define XMR_CRC_VAR_KERNEL(NC, INJ)                                                                      \
    extern "C" __global__ void __launch_bounds__(XMR_CTA_THREADS)                                        \
    xmr_crc16_var_inj##INJ##_nc##NC(const __grid_constant__ xmr_args a) {                                \
        xmr::crc16_var_body<NC, INJ != 0>(a);                                                            \
    }
#define XMR_QSORT_VAR_KERNEL(NC, INJ)                                                                    \
    extern "C" __global__ void __launch_bounds__(XMR_QSORT_THREADS)                                      \
    xmr_qsort_var_inj##INJ##_nc##NC(const __grid_constant__ xmr_args a) {                                \
        xmr::qsort_var_body<NC, INJ != 0>(a);                                                            \
    }
XMR_SHA_VAR_KERNEL(1, 0) XMR_SHA_VAR_KERNEL(2, 0) XMR_SHA_VAR_KERNEL(3, 0)
XMR_SHA_VAR_KERNEL(1, 1) XMR_SHA_VAR_KERNEL(2, 1) XMR_SHA_VAR_KERNEL(3, 1)
XMR_CRC_VAR_KERNEL(1, 0) XMR_CRC_VAR_KERNEL(2, 0) XMR_CRC_VAR_KERNEL(3, 0)
XMR_CRC_VAR_KERNEL(1, 1) XMR_CRC_VAR_KERNEL(2, 1) XMR_CRC_VAR_KERNEL(3, 1)
XMR_QSORT_VAR_KERNEL(1, 0) XMR_QSORT_VAR_KERNEL(2, 0) XMR_QSORT_VAR_KERNEL(3, 0)
XMR_QSORT_VAR_KERNEL(1, 1) XMR_QSORT_VAR_KERNEL(2, 1) XMR_QSORT_VAR_KERNEL(3, 1)
