// xmr_crc16.cuh -- protected CCITT CRC-16 (tests/crc16/crc16.c:21-31 of byuccl/coast)
//
// Unit = one message of unit_bytes (1..255, `unsigned char length` :21) -> u16.  SoR exit = the
// `ret i16` (:30): ONE u16 vote per unit.  Fault sites: s < L: `crc` after byte s (16 bits);
// L <= s < 2L: data byte s-L as loaded by the replica (8 bits).
#pragma once
#include "xmr_common.cuh"

namespace xmr {

// one byte of crc16.c:26-28 on 32-bit registers with the reference's u8/u16 truncations
__device__ __forceinline__ uint32_t crc16_step(uint32_t crc, uint32_t b) {
    uint32_t x = ((crc >> 8) ^ b) & 0xFFu;        // x = crc >> 8 ^ *data_p++   (u8)
    x ^= x >> 4;                                  // x ^= x >> 4
    return ((crc << 8) ^ (x << 12) ^ (x << 5) ^ x) & 0xFFFFu;   // (u16)
}

template <int NC>
__device__ __forceinline__ void crc_vote_store(uint32_t crc, uint16_t* out, unsigned long long local, unsigned long long gunit,
                                               bool valid, int lane, uint32_t flags, Tally& tally) {
    Voted v = vote_u32<NC, 4>(crc, flags & COAST_F_MAJORITY_VOTER);   // one element (the u16 lives alone in the register)
    if (valid && Lanes<NC>::voter(lane)) {
        out[local] = (uint16_t)v.vote;
        tally.unit_exit<NC>(v.bad, 1u, flags, gunit);
    }
}

// ---- table kernel geometry (unit_bytes == 64) -----------------------------------------------------
// The arithmetic byte step costs ~10.6 integer instructions; r01 ncu showed the kernel issue-bound on them.  The TMA
// kernel uses the table form instead:  T[x] = crc16_step(0, x)  (the (crc << 8) term is 0), so
//     crc' = ((crc & 0xFF) << 8) ^ T[(crc >> 8) ^ b]
// With t_i = T[x_i] the state never has to be assembled:  hi_i = lo_(i-1) ^ t_i.hi,  lo_i = t_i.lo,  so
//     x_(i+1) = hi_i ^ b_(i+1) = t_(i-1).lo ^ t_i.hi ^ b_(i+1)                       (ONE 3-input LOP3)
// provided the three bytes sit at the same byte position p of their registers.  b_(i+1) sits at p = (i+1) & 3 of its
// message word, so step i reads a table word with .hi at byte (i+1)&3 and .lo at byte (i+2)&3:
//     even steps: W1 = [lo, hi, lo, hi]   (bytes 0..3)        odd steps: W2 = [hi, lo, hi, lo]
// Row x of the table is 256 B: W1[x] replicated over the 32 lanes, then W2[x] replicated over the 32 lanes (bank = lane:
// no conflicts whatever the data).  The table sits on a 64 KiB boundary of the shared window, so the lookup address is
// ONE byte-permute that also picks byte p:  addr = PRMT(v, lane base) -- as in the AES kernel.
// Per byte: LOP3 + PRMT + LDS (r01 history: arithmetic 10.6 ALU -> combined-state table 9 -> split state 3.75 + LDS ->
// this form 2 + LDS; 0.394 -> 0.244 -> see profiles/ for the current time of 2^22 TMR messages).
// 64 KiB of table leaves one CTA per SM, so the CTA is 1024 threads (768 for the unprotected run, whose 64 B x 1024
// tile ring would not fit next to the table).
constexpr uint32_t CRC_TAB = XMR_CRC_TAB, CRC_RING = XMR_CRC_RING;
static_assert(CRC_TAB + 256u * 64u * 4u <= CRC_RING, "the table ends below the ring");
template <int NC> struct CrcGeom {
    static constexpr int THREADS = (int)xmr_crc_threads(NC);
    static constexpr int WARPS = THREADS / 32;
    static constexpr int TU = WARPS * Lanes<NC>::kUnitsPerWarp;
};
template <int OFF>
__device__ __forceinline__ uint32_t crc_lds32(uint32_t saddr) { uint32_t v; asm volatile("ld.shared.u32 %0, [%1+%2];" : "=r"(v) : "r"(saddr), "n"(OFF)); return v; }

struct CrcWidth { uint32_t len; __device__ uint32_t operator()(uint32_t site) const { return site < len ? 16u : 8u; } };

// Fast path: unit_bytes == 64.  A ring stage holds one tile of WARPS*(32/NC) messages; every lane runs CRC_J = 2
// messages at once (one from each stage) because a single chain LOP3 -> PRMT -> LDS -> LOP3 is latency-bound even at 32
// warps per SM (r01: 2.8 cycles per warp byte-step with one chain; the issue and LDS limits are ~1.2 and ~1.0).  The two
// stages are refilled right after the words are in registers, so the TMA latency hides behind the 64-step loop.
//
// Injection: `crc` is used by the next step only through x = (crc >> 8) ^ b, so a flip of crc bit 8+k after byte s IS a
// flip of bit k of data byte s+1 as that replica sees it, and a flip of bit k < 8 (which becomes bit 8+k one step later)
// IS a flip of bit k of data byte s+2; flips falling off the end land in the returned crc.  The faulted replica
// therefore XORs one mask into one of its 16 private message words (or into the result) instead of testing the site
// index at all 128 hook points; the voted output and the counters are bit-identical to the hook-per-site form (oracle
// parity tests).
constexpr int CRC_J = 2;
template <int NC, bool INJECT>
__device__ __forceinline__ void crc16_b64_body(const xmr_args& a, const CUtensorMap* tmap) {
    using G = CrcGeom<NC>;
    constexpr int UPW = Lanes<NC>::kUnitsPerWarp;
    constexpr int TU = G::TU;
    static_assert(XMR_STAGES == CRC_J, "one ring stage per in-flight message of a lane");
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    using Ring = TileRing<TU, 64>;
    static_assert(TU == xmr_crc_tile_rows(NC) && CRC_RING + Ring::SMEM_BYTES <= xmr_crc_smem(NC), "ring fits the launch's shared memory");
    const uint32_t win = smem_u32(smem_raw);                    // shared-window address of the dynamic region
    Ring ring;
    ring.init(smem_raw + (CRC_RING - win), tmap);
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    {
        uint32_t* tab = reinterpret_cast<uint32_t*>(smem_raw + (CRC_TAB - win));
        for (int i = tid; i < 256 * 32; i += G::THREADS) {
            const uint32_t x = (uint32_t)i >> 5;
            const uint32_t t = crc16_step(0u, x);               // the reference's own byte step fills the table
            const uint32_t h = t >> 8, l = t & 0xFFu;
            tab[x * 64u + ((uint32_t)i & 31u)] = l | (h << 8) | (l << 16) | (h << 24);         // W1: even steps
            tab[x * 64u + 32u + ((uint32_t)i & 31u)] = h | (l << 8) | (h << 16) | (l << 24);   // W2: odd steps
        }
    }
    __syncthreads();
    const uint32_t lb = CRC_TAB + 4u * (uint32_t)lane;
    const int r = Lanes<NC>::replica(lane);
    const int ul = warp * UPW + Lanes<NC>::unit(lane);
    const int sw = (ul >> 1) & 3;
    const uint32_t n_pairs = (a.n_tiles + CRC_J - 1u) / CRC_J;  // a tile past the end is zero-filled by TMA and masked by `valid`
    uint32_t pair = blockIdx.x;
    if (pair < n_pairs) {
#pragma unroll
        for (int j = 0; j < CRC_J; ++j) ring.issue(j, pair * CRC_J + j);
    }
    Tally tally(a);
    uint32_t it = 0;
    for (; pair < n_pairs; pair += gridDim.x, ++it) {
        uint32_t w[CRC_J][16];
#pragma unroll
        for (int j = 0; j < CRC_J; ++j) {
            mbar_wait(&ring.full[j], it & 1u);
            const uint8_t* row = ring.tiles + j * Ring::STAGE_STRIDE + ul * 64;
#pragma unroll
            for (int c = 0; c < 4; ++c) {
                uint4 q = *reinterpret_cast<const uint4*>(row + ((c ^ sw) << 4));
                w[j][4 * c] = q.x; w[j][4 * c + 1] = q.y; w[j][4 * c + 2] = q.z; w[j][4 * c + 3] = q.w;
            }
        }
        __syncthreads();
        const uint32_t next = pair + gridDim.x;
        if (next < n_pairs) {
#pragma unroll
            for (int j = 0; j < CRC_J; ++j) ring.issue(j, next * CRC_J + j);
        }
        unsigned long long local[CRC_J];
        bool valid[CRC_J];
        uint32_t ffin[CRC_J];
#pragma unroll
        for (int j = 0; j < CRC_J; ++j) {
            local[j] = ((unsigned long long)pair * CRC_J + j) * TU + ul;
            valid[j] = local[j] < a.n_units;
            ffin[j] = 0u;
            if (INJECT) {
                Fault f = fault_for_unit(a, NC, valid[j] ? local[j] : 0ull, CrcWidth{64u});
                uint32_t fw = 0xFFFFFFFFu, fwm = 0u;
                if (f.active && valid[j]) {
                    if (Lanes<NC>::voter(lane)) tally.injected++;
                    if ((int)f.replica == r) {
                        const bool data = f.site >= 64u, high = f.bit >= 8u;
                        const uint32_t pos = data ? f.site - 64u : f.site + (high ? 1u : 2u);   // data byte that carries the flip
                        const uint32_t m8 = 1u << (high ? f.bit - 8u : f.bit);
                        if (pos < 64u) { fw = pos >> 2; fwm = m8 << (8u * (pos & 3u)); }
                        else ffin[j] = high ? (1u << f.bit) : (pos == 64u ? (m8 << 8) : m8);    // fell off the end: in the result
                    }
                }
#pragma unroll
                for (int k = 0; k < 16; ++k) w[j][k] ^= (fw == (uint32_t)k) ? fwm : 0u;
            }
        }
        // crc = 0xFFFF (:23) as the two table words "before" byte 0: t_(-1) = {hi 0xFF @ byte 0, lo 0xFF @ byte 1}, t_(-2) = 0
        uint32_t t1[CRC_J], t2[CRC_J];
#pragma unroll
        for (int j = 0; j < CRC_J; ++j) { t1[j] = 0xFFFFu; t2[j] = 0u; }
#pragma unroll
        for (int i = 0; i < 64; ++i) {                         // :25
#pragma unroll
            for (int j = 0; j < CRC_J; ++j) {
                const uint32_t v = t2[j] ^ t1[j] ^ w[j][i >> 2];                   // x = crc >> 8 ^ *data_p++ at byte i & 3
                const uint32_t addr = __byte_perm(v, lb, 0x7604u | ((uint32_t)(i & 3) << 4));
                t2[j] = t1[j];
                t1[j] = (i & 1) ? crc_lds32<128>(addr) : crc_lds32<0>(addr);
            }
        }
#pragma unroll
        for (int j = 0; j < CRC_J; ++j) {
            // hi_63 = t_62.lo ^ t_63.hi (both at byte 0), lo_63 = t_63.lo (byte 1)
            const uint32_t crc = ((((t2[j] ^ t1[j]) & 0xFFu) << 8) | ((t1[j] >> 8) & 0xFFu)) ^ ffin[j];
            crc_vote_store<NC>(crc, static_cast<uint16_t*>(a.out), local[j], a.unit_base + local[j], valid[j], lane, a.flags, tally);
        }
    }
    tally.flush(a.counters);
}

// General path: any length 1..255, bytes read straight from global memory (word loads when every message is 4-byte
// aligned).  Table form of the byte step (r02; the r01 general path ran the 10.6-instruction arithmetic step):
//     crc' = ((crc << 8) & 0xFFFF) ^ T[(crc >> 8) ^ b],   T[x] = crc16_step(0, x)
// with T replicated over the 32 lanes in shared memory (bank = lane: conflict-free whatever the data).
template <int NC, bool INJECT>
__device__ __forceinline__ void crc16_gen_body(const xmr_args& a) {
    constexpr int UPW = Lanes<NC>::kUnitsPerWarp;
    __shared__ uint32_t tab[256 * 32];
    for (int i = threadIdx.x; i < 256 * 32; i += blockDim.x) tab[i] = crc16_step(0u, (uint32_t)i >> 5);   // the reference's own byte step fills the table
    __syncthreads();
    const int lane = threadIdx.x & 31;
    const uint32_t* const tl = tab + lane;
    const bool words = ((reinterpret_cast<uintptr_t>(a.in) | a.unit_bytes) & 3u) == 0;
    const int r = Lanes<NC>::replica(lane);
    const unsigned long long gwarp = ((unsigned long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const unsigned long long nwarps = ((unsigned long long)gridDim.x * blockDim.x) >> 5;
    const unsigned long long n_wtiles = (a.n_units + UPW - 1) / UPW;
    const uint32_t len = a.unit_bytes;
    Tally tally(a);
    for (unsigned long long wt = gwarp; wt < n_wtiles; wt += nwarps) {
        const unsigned long long local = wt * UPW + Lanes<NC>::unit(lane);
        const bool valid = local < a.n_units;
        const uint8_t* msg = static_cast<const uint8_t*>(a.in) + (valid ? local : 0ull) * len;
        uint32_t fsite = 0xFFFFFFFFu, fmask = 0u;
        if (INJECT) {
            Fault f = fault_for_unit(a, NC, valid ? local : 0ull, CrcWidth{len});
            if (f.active && valid) {
                if (Lanes<NC>::voter(lane)) tally.injected++;
                if ((int)f.replica == r) { fsite = f.site; fmask = 1u << f.bit; }
            }
        }
        uint32_t crc = 0xFFFFu;
        if (!(a.flags & XMR_F_STORE_VOTES)) {
            uint32_t w = 0;
            for (uint32_t i = 0; i < len; ++i) {
                if (words) { if ((i & 3u) == 0) w = __ldg(reinterpret_cast<const uint32_t*>(msg + i)); }
                uint32_t b = words ? (w >> (8u * (i & 3u))) & 0xFFu : (uint32_t)__ldg(msg + i);
                if (INJECT && fsite == len + i) b ^= fmask;
                crc = ((crc << 8) & 0xFFFFu) ^ tl[(((crc >> 8) ^ b) & 0xFFu) << 5];
                if (INJECT && fsite == i) crc ^= fmask;
            }
            crc_vote_store<NC>(crc, static_cast<uint16_t*>(a.out), local, a.unit_base + local, valid, lane, a.flags, tally);
        } else {
            // -storeDataSync / -noMemReplication: the three assignments of the loop body are voted (crc16.c:26-28), the
            // replicas continue with the voted value; 3 votes per byte + the SoR exit
            const bool majority = a.flags & COAST_F_MAJORITY_VOTER;
            uint32_t bad = 0;
            for (uint32_t i = 0; i < len; ++i) {
                uint32_t b = __ldg(msg + i);
                if (INJECT && fsite == len + i) b ^= fmask;
                uint32_t x = ((crc >> 8) ^ b) & 0xFFu;                              // :26
                bad += store_vote<NC>(x, lane, majority);
                x = (x ^ (x >> 4)) & 0xFFu;                                         // :27
                bad += store_vote<NC>(x, lane, majority);
                crc = ((crc << 8) ^ (x << 12) ^ (x << 5) ^ x) & 0xFFFFu;            // :28
                bad += store_vote<NC>(crc, lane, majority);
                if (INJECT && fsite == i) crc ^= fmask;
            }
            bad += store_vote<NC>(crc, lane, majority);                             // :30
            if (valid && Lanes<NC>::voter(lane)) {
                static_cast<uint16_t*>(a.out)[local] = (uint16_t)crc;
                tally.unit_exit<NC>(bad, 3u * len + 1u, a.flags, a.unit_base + local);
            }
        }
    }
    tally.flush(a.counters);
}

}  // namespace xmr

#define XMR_CRC_B64_KERNEL(NC, INJ)                                                                      \
    extern "C" __global__ void __launch_bounds__(xmr::CrcGeom<NC>::THREADS)                              \
    xmr_crc16_b64_nc##NC##_inj##INJ(const __grid_constant__ xmr_args a, const __grid_constant__ CUtensorMap tmap) { \
        xmr::crc16_b64_body<NC, INJ != 0>(a, &tmap);                                                     \
    }
#define XMR_CRC_GEN_KERNEL(NC, INJ)                                                                      \
    extern "C" __global__ void __launch_bounds__(XMR_CTA_THREADS)                                        \
    xmr_crc16_gen_nc##NC##_inj##INJ(const __grid_constant__ xmr_args a) {                                \
        xmr::crc16_gen_body<NC, INJ != 0>(a);                                                            \
    }
XMR_CRC_B64_KERNEL(1, 0) XMR_CRC_B64_KERNEL(2, 0) XMR_CRC_B64_KERNEL(3, 0)
XMR_CRC_B64_KERNEL(1, 1) XMR_CRC_B64_KERNEL(2, 1) XMR_CRC_B64_KERNEL(3, 1)
XMR_CRC_GEN_KERNEL(1, 0) XMR_CRC_GEN_KERNEL(2, 0) XMR_CRC_GEN_KERNEL(3, 0)
XMR_CRC_GEN_KERNEL(1, 1) XMR_CRC_GEN_KERNEL(2, 1) XMR_CRC_GEN_KERNEL(3, 1)
