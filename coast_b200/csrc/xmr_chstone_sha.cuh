// xmr_chstone_sha.cuh -- protected CHStone `sha` (tests/chstone/sha/sha.c of byuccl/coast; SURVEY.md 8f-4)
//
// The CHStone variant of the NIST hash: no rotate in the W expansion (USE_MODIFIED_SHA undefined, sha.c:101), words
// loaded LITTLE-endian by the benchmark's own memcpy (:71-90), and a final block whose 0x80 marker is written at a
// WORD index computed from a BYTE count (:167-168).  Unit = one stream of unit_bytes (a multiple of 64, < 2^29):
// sha_init (:131-139), one sha_transform (:93-127) per 64-byte block (sha_update :149-154), and sha_final's block
// {0x80, 0 x 13, hi = 0, lo = 8 * unit_bytes} (:168-178).  SoR exit = the five LONG words of sha_info_digest
// (sha.h:38, compared in sha_driver.c:59): FIVE u32 votes per unit.
//
// A stream is a serial chain of unit_bytes/64 + 1 compressions, so one lane walks one replica of one stream; replicas
// sit on adjacent lanes (Lanes<NC>).  The next block's 16 words are loaded (4 x LDG.128, native byte order -- the
// little-endian pack is free) before the current block's 80 rounds run.
//
// Fault sites per compression c (site = 421*c + s):  s < 16: W[s] as loaded;  16 <= s < 416: working variable
// (s-16)%5 of (A,B,C,D,E) before round (s-16)/5;  416 <= s < 421: sha_info_digest[s-416] after the final add.
// Only the ONE compression that holds a lane's fault runs the hooked (rolled, W[80] in local memory) transform; all
// others run the unrolled one with a 16-word rolling schedule window.
#pragma once
#include "xmr_common.cuh"

namespace xmr {

constexpr uint32_t CHS_SITES_PER_BLOCK = 421u;

__device__ __forceinline__ uint32_t chs_rotl(uint32_t v, int n) { return __funnelshift_l(v, v, n); }

template <int T> __device__ __forceinline__ uint32_t chs_f(uint32_t B, uint32_t C, uint32_t D) {
    if (T < 20) return (B & C) | (~B & D);                 // f1 :30
    if (T < 40) return B ^ C ^ D;                          // f2 :31
    if (T < 60) return (B & C) | (B & D) | (C & D);        // f3 :32
    return B ^ C ^ D;                                      // f4 :33
}
template <int T> __device__ __forceinline__ uint32_t chs_k() {
    return T < 20 ? 0x5a827999u : T < 40 ? 0x6ed9eba1u : T < 60 ? 0x8f1bbcdcu : 0xca62c1d6u;   // :35-38
}

template <int T>
__device__ __forceinline__ void chs_rounds(uint32_t (&W)[16], uint32_t& A, uint32_t& B, uint32_t& C, uint32_t& D, uint32_t& E) {
    if constexpr (T < 80) {
        uint32_t w;
        if (T < 16) w = W[T];                                                            // :97-99
        else { w = W[(T - 3) & 15] ^ W[(T - 8) & 15] ^ W[(T - 14) & 15] ^ W[T & 15]; W[T & 15] = w; }   // :100-102
        const uint32_t temp = chs_rotl(A, 5) + chs_f<T>(B, C, D) + E + w + chs_k<T>();   // FUNC :47-53
        E = D; D = C; C = chs_rotl(B, 30); B = A; A = temp;
        chs_rounds<T + 1>(W, A, B, C, D, E);
    }
}

__device__ __forceinline__ void chs_transform(uint32_t (&dig)[5], uint32_t (&W)[16]) {
    uint32_t A = dig[0], B = dig[1], C = dig[2], D = dig[3], E = dig[4];                // :103-107
    chs_rounds<0>(W, A, B, C, D, E);
    dig[0] += A; dig[1] += B; dig[2] += C; dig[3] += D; dig[4] += E;                     // :122-126
}

// the compression that carries a fault: same arithmetic, every site hooked, loops rolled
__device__ __noinline__ void chs_transform_faulted(uint32_t* dig, const uint32_t* w16, uint32_t s, uint32_t mask) {
    uint32_t W[80], v[5];
#pragma unroll 1
    for (int i = 0; i < 16; ++i) W[i] = w16[i];
    if (s < 16u) W[s] ^= mask;
#pragma unroll 1
    for (int i = 16; i < 80; ++i) W[i] = W[i - 3] ^ W[i - 8] ^ W[i - 14] ^ W[i - 16];
#pragma unroll
    for (int i = 0; i < 5; ++i) v[i] = dig[i];
#pragma unroll 1
    for (uint32_t t = 0; t < 80u; ++t) {
        if (s >= 16u && s < 416u && (s - 16u) / 5u == t) {
            const uint32_t k = (s - 16u) % 5u;
#pragma unroll
            for (int j = 0; j < 5; ++j) v[j] ^= (k == (uint32_t)j) ? mask : 0u;
        }
        const uint32_t A = v[0], B = v[1], C = v[2], D = v[3], E = v[4];
        uint32_t fn, k;
        if (t < 20u)      { fn = (B & C) | (~B & D);          k = 0x5a827999u; }
        else if (t < 40u) { fn = B ^ C ^ D;                   k = 0x6ed9eba1u; }
        else if (t < 60u) { fn = (B & C) | (B & D) | (C & D); k = 0x8f1bbcdcu; }
        else              { fn = B ^ C ^ D;                   k = 0xca62c1d6u; }
        const uint32_t temp = chs_rotl(A, 5) + fn + E + W[t] + k;
        v[4] = D; v[3] = C; v[2] = chs_rotl(B, 30); v[1] = A; v[0] = temp;
    }
#pragma unroll
    for (int i = 0; i < 5; ++i) dig[i] += v[i];
    if (s >= 416u && s < 421u) {
#pragma unroll
        for (int j = 0; j < 5; ++j) dig[j] ^= (s - 416u == (uint32_t)j) ? mask : 0u;
    }
}

template <int NC, bool INJECT>
__device__ __forceinline__ void chsha_body(const xmr_args& a) {
    constexpr int UPW = Lanes<NC>::kUnitsPerWarp;
    const int lane = threadIdx.x & 31;
    const int r = Lanes<NC>::replica(lane);
    const unsigned long long gwarp = ((unsigned long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const unsigned long long nwarps = ((unsigned long long)gridDim.x * blockDim.x) >> 5;
    const unsigned long long n_wtiles = (a.n_units + UPW - 1) / UPW;
    const uint32_t len = a.unit_bytes;
    const uint32_t nblk = len >> 6;                            // data blocks; the final block is compression #nblk
    const bool majority = a.flags & COAST_F_MAJORITY_VOTER;
    Tally tally(a);
    for (unsigned long long wt = gwarp; wt < n_wtiles; wt += nwarps) {
        const unsigned long long local = wt * UPW + Lanes<NC>::unit(lane);
        const bool valid = local < a.n_units;
        const unsigned long long gunit = a.unit_base + local;
        const uint4* msg = reinterpret_cast<const uint4*>(static_cast<const uint8_t*>(a.in) + (valid ? local : 0ull) * len);
        uint32_t fblk = 0xFFFFFFFFu, fs = 0u, fmask = 0u;
        if (INJECT) {
            Fault f = fault_for_unit(a, NC, valid ? local : 0ull, [](uint32_t) { return 32u; });
            if (f.active && valid) {
                if (Lanes<NC>::voter(lane)) tally.injected++;
                if ((int)f.replica == r) { fmask = 1u << f.bit; fblk = f.site / CHS_SITES_PER_BLOCK; fs = f.site % CHS_SITES_PER_BLOCK; }
            }
        }
        uint32_t dig[5] = { 0x67452301u, 0xefcdab89u, 0x98badcfeu, 0x10325476u, 0xc3d2e1f0u };   // sha_init :132-136
        uint4 q[4];
#pragma unroll
        for (int c = 0; c < 4; ++c) q[c] = nblk ? __ldg(msg + c) : make_uint4(0u, 0u, 0u, 0u);
        for (uint32_t blk = 0; blk <= nblk; ++blk) {
            uint32_t W[16];
            if (blk < nblk) {                                  // sha_update :149-154 (memcpy :78-89 = native little-endian words)
#pragma unroll
                for (int c = 0; c < 4; ++c) { W[4 * c] = q[c].x; W[4 * c + 1] = q[c].y; W[4 * c + 2] = q[c].z; W[4 * c + 3] = q[c].w; }
                if (blk + 1u < nblk) {
#pragma unroll
                    for (int c = 0; c < 4; ++c) q[c] = __ldg(msg + 4u * (blk + 1u) + c);
                }
            } else {                                           // sha_final :168-177 with count == 0
#pragma unroll
                for (int i = 0; i < 16; ++i) W[i] = 0u;
                W[0] = 0x80u; W[15] = len << 3;
            }
            if (INJECT && blk == fblk) chs_transform_faulted(dig, W, fs, fmask);
            else chs_transform(dig, W);
        }
        uint32_t o[5], bad = 0;
#pragma unroll
        for (int i = 0; i < 5; ++i) { Voted v = vote_u32<NC, 4>(dig[i], majority); o[i] = v.vote; bad += v.bad; }
        if (valid && Lanes<NC>::voter(lane)) {
            uint32_t* dst = static_cast<uint32_t*>(a.out) + local * 5ull;
#pragma unroll
            for (int i = 0; i < 5; ++i) dst[i] = o[i];
            tally.unit_exit<NC>(bad, 5u, a.flags, gunit);
        }
    }
    tally.flush(a.counters);
}

}  // namespace xmr

#define XMR_CHSHA_KERNEL(NC, INJ)                                                                        \
    extern "C" __global__ void __launch_bounds__(XMR_CTA_THREADS)                                        \
    xmr_chsha_nc##NC##_inj##INJ(const __grid_constant__ xmr_args a) {                                    \
        xmr::chsha_body<NC, INJ != 0>(a);                                                                \
    }
XMR_CHSHA_KERNEL(1, 0) XMR_CHSHA_KERNEL(2, 0) XMR_CHSHA_KERNEL(3, 0)
XMR_CHSHA_KERNEL(1, 1) XMR_CHSHA_KERNEL(2, 1) XMR_CHSHA_KERNEL(3, 1)
