// xmr_sha256.cuh -- protected SHA-256 (tests/sha256_common/sha256_common_tmr.c:28-180 of byuccl/coast)
//
// Unit = one message of `unit_bytes` bytes -> 32 digest bytes.
//   sha256_transform  (:28-98)   -> sha_compress<INJECT>()
//   sha256_hash       (:101-180) -> message feed / 0x80 padding / 64-bit big-endian bit length /
//                                   big-endian digest bytes, in xmr_sha256_b64 (len == 64, the
//                                   BASELINE configs 2 and 5) and xmr_sha256_gen (any length).
// SoR exit = the 32 u8 stores `hash[i] = ...` (:169-178): 32 votes per unit, voted 4-at-a-time
// with byte-granular compare/select so counts equal 32 separate u8 votes.
//
// HBM traffic: the message tile is brought in ONCE by TMA (cp.async.bulk.tensor, 64B-swizzled
// so the per-lane 16-byte reads are bank-conflict free); the NC replica lanes of a unit read the
// same shared-memory bytes (broadcast) -- "-noMemReplication for inputs only" (passes.rst:331).
// Only the voter lane stores the digest: one voted output.
#pragma once
#include "xmr_common.cuh"

namespace xmr {

// K as compile-time immediates for the fully unrolled rounds
__device__ __forceinline__ constexpr uint32_t sha_k(int i) {
    constexpr uint32_t K[64] = {
        0x428a2f98u, 0x71374491u, 0xb5c0fbcfu, 0xe9b5dba5u, 0x3956c25bu, 0x59f111f1u, 0x923f82a4u, 0xab1c5ed5u,
        0xd807aa98u, 0x12835b01u, 0x243185beu, 0x550c7dc3u, 0x72be5d74u, 0x80deb1feu, 0x9bdc06a7u, 0xc19bf174u,
        0xe49b69c1u, 0xefbe4786u, 0x0fc19dc6u, 0x240ca1ccu, 0x2de92c6fu, 0x4a7484aau, 0x5cb0a9dcu, 0x76f988dau,
        0x983e5152u, 0xa831c66du, 0xb00327c8u, 0xbf597fc7u, 0xc6e00bf3u, 0xd5a79147u, 0x06ca6351u, 0x14292967u,
        0x27b70a85u, 0x2e1b2138u, 0x4d2c6dfcu, 0x53380d13u, 0x650a7354u, 0x766a0abbu, 0x81c2c92eu, 0x92722c85u,
        0xa2bfe8a1u, 0xa81a664bu, 0xc24b8b70u, 0xc76c51a3u, 0xd192e819u, 0xd6990624u, 0xf40e3585u, 0x106aa070u,
        0x19a4c116u, 0x1e376c08u, 0x2748774cu, 0x34b0bcb5u, 0x391c0cb3u, 0x4ed8aa4au, 0x5b9cca4fu, 0x682e6ff3u,
        0x748f82eeu, 0x78a5636fu, 0x84c87814u, 0x8cc70208u, 0x90befffau, 0xa4506cebu, 0xbef9a3f7u, 0xc67178f2u};
    return K[i];
}

constexpr uint32_t SHA_SITES_PER_BLOCK = 536u;   // 16 m[] + 64 rounds x 8 working vars + 8 ctx_state

__device__ __forceinline__ uint32_t rotr(uint32_t v, int n) { return __funnelshift_r(v, v, n); }
__device__ __forceinline__ uint32_t bswap(uint32_t v) { return __byte_perm(v, 0u, 0x0123u); }

// The compression is bound by ALU-pipe issue: its rotations, XORs and additions all go to the ALU pipe, which takes one warp
// instruction every 2 cycles per SM sub-partition, while the IMAD pipe beside it idles.  Additions are issued there instead as
// x * 1 + y (DESIGN.md §5.0).  The 1 lives in the constant bank: IMAD reads it from a uniform register, costing no register, and
// ptxas, which cannot know its value, cannot turn the product back into an IADD3.  The shifts and rotations stay on the ALU
// pipe: their multiply forms need IMAD.HI, which runs at half rate.
__constant__ uint32_t sha_one = 1u;

__device__ __forceinline__ uint32_t add_imad(uint32_t x, uint32_t y) {
    uint32_t d;
    asm("mad.lo.u32 %0, %1, %2, %3;" : "=r"(d) : "r"(x), "r"(sha_one), "r"(y));
    return d;
}

// x + k for a compile-time k (the padding block's K + W), as IMAD one, k, x.  The 1 has to be in a per-thread register here
// (an IMAD with an immediate takes no constant-bank or uniform operand besides it), so it is a constant of its own: were it
// sha_one, ptxas would read that register in every add_imad as well, a third register source per IMAD where the uniform
// register serves, and the kernel runs 9% slower so (DESIGN.md §5.0).  The alignment keeps it out of sha_one's 8 bytes, which
// ptxas would otherwise fetch together with one LDC.64 into registers.
__constant__ __align__(16) uint32_t sha_one_imm = 1u;

__device__ __forceinline__ uint32_t add_imad_imm(uint32_t x, uint32_t k) {
    uint32_t d;
    asm("mad.lo.u32 %0, %1, %2, %3;" : "=r"(d) : "r"(sha_one_imm), "r"(k), "r"(x));
    return d;
}

// One compression.  m[0..15] holds the big-endian-packed block (:34-40) and is used as the rolling
// 16-word schedule window (:42-58).  `fs`/`fmask`: fault site within THIS block (>= 536 = none).
// CONST_M: m[] holds compile-time constants (the padding block of a 64-byte message); its schedule is written with plain
// additions so that it folds away, which add_imad would prevent.
template <bool INJECT, bool CONST_M = false>
__device__ __forceinline__ void sha_compress(uint32_t (&st)[8], uint32_t (&m)[16], uint32_t fs, uint32_t fmask) {
    if (INJECT && fs < 16u) {
#pragma unroll
        for (int i = 0; i < 16; ++i) m[i] ^= fs == (uint32_t)i ? fmask : 0u;
    }
    uint32_t a = st[0], b = st[1], c = st[2], d = st[3], e = st[4], f = st[5], g = st[6], h = st[7];
    const uint32_t ft = INJECT ? ((fs - 16u) >> 3) : 0u;      // round of the fault (valid when 16 <= fs < 528)
    const uint32_t fv = INJECT ? ((fs - 16u) & 7u) : 0u;
    const bool fround = INJECT && fs >= 16u && fs < 528u;
#pragma unroll
    for (int t = 0; t < 64; ++t) {
        if (t >= 16) {                                         // :42-58
            uint32_t w2 = m[(t - 2) & 15], w15 = m[(t - 15) & 15];
            uint32_t s1 = rotr(w2, 17) ^ rotr(w2, 19) ^ (w2 >> 10);
            uint32_t s0 = rotr(w15, 7) ^ rotr(w15, 18) ^ (w15 >> 3);
            m[t & 15] = CONST_M ? s1 + m[(t - 7) & 15] + s0 + m[t & 15]
                                : add_imad(s1, add_imad(s0, add_imad(m[(t - 7) & 15], m[t & 15])));
        }
        if (INJECT && fround && ft == (uint32_t)t) {
            a ^= fv == 0 ? fmask : 0u; b ^= fv == 1 ? fmask : 0u; c ^= fv == 2 ? fmask : 0u; d ^= fv == 3 ? fmask : 0u;
            e ^= fv == 4 ? fmask : 0u; f ^= fv == 5 ? fmask : 0u; g ^= fv == 6 ? fmask : 0u; h ^= fv == 7 ? fmask : 0u;
        }
        uint32_t ep0 = rotr(a, 2) ^ rotr(a, 13) ^ rotr(a, 22);  // :70-72
        uint32_t ep1 = rotr(e, 6) ^ rotr(e, 11) ^ rotr(e, 25);  // :73-75
        uint32_t ch = (e & f) ^ (~e & g);                       // :76
        uint32_t maj = (a & b) ^ (a & c) ^ (b & c);             // :77
        const uint32_t hkw = CONST_M ? add_imad_imm(h, sha_k(t) + m[t & 15]) : add_imad(h, sha_k(t) + m[t & 15]);   // K + W
        uint32_t t1 = add_imad(ep1, add_imad(ch, hkw));         // :78
        uint32_t t2 = add_imad(ep0, maj);                       // :79
        h = g; g = f; f = e; e = add_imad(d, t1); d = c; c = b; b = a; a = add_imad(t1, t2);   // :80-87
    }
    st[0] += a; st[1] += b; st[2] += c; st[3] += d; st[4] += e; st[5] += f; st[6] += g; st[7] += h;   // :90-97
    if (INJECT && fs >= 528u && fs < 536u) {
#pragma unroll
        for (int i = 0; i < 8; ++i) st[i] ^= fs - 528u == (uint32_t)i ? fmask : 0u;
    }
}

// -storeDataSync / -noMemReplication (coast_rt.h "in-loop store votes"): the same compression with EVERY assignment to a data
// variable voted and, under TMR, all replicas continuing with the voted value -- m[i] (:34-58), a..h = ctx_state (:60-67),
// t1, t2, h, g, f, e, d, c, b, a per round (:78-87), ctx_state += (:90-97): 720 votes.  The schedule is computed on the fly as
// in sha_compress; every vote sees the operands it would see in the reference's order (each voted value re-converges).
// Returns the number of votes at which the copies disagreed.  All 32 lanes must call.
template <int NC, bool INJECT>
__device__ __forceinline__ uint32_t sha_compress_sv(uint32_t (&st)[8], uint32_t (&m)[16], uint32_t fs, uint32_t fmask, int lane, bool majority) {
    uint32_t bad = 0;
#define SV(x) bad += store_vote<NC>(x, lane, majority)
#pragma unroll
    for (int i = 0; i < 16; ++i) { SV(m[i]); if (INJECT) m[i] ^= fs == (uint32_t)i ? fmask : 0u; }
    uint32_t v[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) { v[i] = st[i]; SV(v[i]); }
    uint32_t a = v[0], b = v[1], c = v[2], d = v[3], e = v[4], f = v[5], g = v[6], h = v[7];
    const uint32_t ft = INJECT ? ((fs - 16u) >> 3) : 0u, fv = INJECT ? ((fs - 16u) & 7u) : 0u;
    const bool fround = INJECT && fs >= 16u && fs < 528u;
#pragma unroll 1
    for (int t = 0; t < 64; ++t) {
        if (t >= 16) {
            const uint32_t w2 = m[(t - 2) & 15], w15 = m[(t - 15) & 15];
            uint32_t w = (rotr(w2, 17) ^ rotr(w2, 19) ^ (w2 >> 10)) + m[(t - 7) & 15] + (rotr(w15, 7) ^ rotr(w15, 18) ^ (w15 >> 3)) + m[t & 15];
            SV(w);
            m[t & 15] = w;
        }
        if (INJECT && fround && ft == (uint32_t)t) {
            a ^= fv == 0 ? fmask : 0u; b ^= fv == 1 ? fmask : 0u; c ^= fv == 2 ? fmask : 0u; d ^= fv == 3 ? fmask : 0u;
            e ^= fv == 4 ? fmask : 0u; f ^= fv == 5 ? fmask : 0u; g ^= fv == 6 ? fmask : 0u; h ^= fv == 7 ? fmask : 0u;
        }
        uint32_t t1 = h + (rotr(e, 6) ^ rotr(e, 11) ^ rotr(e, 25)) + ((e & f) ^ (~e & g)) + sha_k(t) + m[t & 15];
        SV(t1);
        uint32_t t2 = (rotr(a, 2) ^ rotr(a, 13) ^ rotr(a, 22)) + ((a & b) ^ (a & c) ^ (b & c));
        SV(t2);
        uint32_t x;
        x = g; SV(x); h = x;
        x = f; SV(x); g = x;
        x = e; SV(x); f = x;
        x = d + t1; SV(x); e = x;
        x = c; SV(x); d = x;
        x = b; SV(x); c = x;
        x = a; SV(x); b = x;
        x = t1 + t2; SV(x); a = x;
    }
    const uint32_t add[8] = {a, b, c, d, e, f, g, h};
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        uint32_t x = st[i] + add[i];
        SV(x);
        st[i] = x;
        if (INJECT) st[i] ^= (fs >= 528u && fs - 528u == (uint32_t)i) ? fmask : 0u;
    }
#undef SV
    return bad;
}

__device__ __forceinline__ void sha_init(uint32_t (&st)[8]) {   // :108-115
    st[0] = 0x6a09e667u; st[1] = 0xbb67ae85u; st[2] = 0x3c6ef372u; st[3] = 0xa54ff53au;
    st[4] = 0x510e527fu; st[5] = 0x9b05688cu; st[6] = 0x1f83d9abu; st[7] = 0x5be0cd19u;
}

// SoR exit: 32 u8 votes (:169-178), one coalesced 32-byte store by the voter lane.
template <int NC>
__device__ __forceinline__ void sha_vote_store(const uint32_t (&st)[8], uint8_t* out, unsigned long long local,
                                               unsigned long long gunit, bool valid, int lane, uint32_t flags, Tally& tally) {
    const bool majority = flags & COAST_F_MAJORITY_VOTER;
    uint32_t o[8], bad = 0;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        Voted v = vote_u32<NC, 1>(st[i], majority);
        o[i] = bswap(v.vote);                       // big-endian digest bytes
        bad += v.bad;
    }
    if (valid && Lanes<NC>::voter(lane)) {
        uint4* dst = reinterpret_cast<uint4*>(out + local * 32ull);
        dst[0] = make_uint4(o[0], o[1], o[2], o[3]);
        dst[1] = make_uint4(o[4], o[5], o[6], o[7]);
        tally.unit_exit<NC>(bad, 32u, flags, gunit);
    }
}

// ---------------------------------------------------------------------------------------------
// Fast path: unit_bytes == 64 (two compressions; the second block is the constant padding block).
// grid = persistent CTAs, 8 warps, tile = 8 * (32/NC) messages staged by TMA, 2-stage ring.
// ---------------------------------------------------------------------------------------------
template <int NC, bool INJECT>
__device__ __forceinline__ void sha256_b64_body(const xmr_args& a, const CUtensorMap* tmap) {
    constexpr int UPW = Lanes<NC>::kUnitsPerWarp;
    constexpr int TU = XMR_WARPS * UPW;                       // units per tile
    static_assert(TU == xmr_sha_tile_rows(NC) && TileRing<TU, 64>::SMEM_BYTES <= xmr_sha_smem(NC), "ring fits the launch's shared memory");
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    TileRing<TU, 64> ring;
    ring.init(smem_raw, tmap);

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int r = Lanes<NC>::replica(lane);
    const int ul = warp * UPW + Lanes<NC>::unit(lane);        // unit within the tile

    const uint32_t n_tiles = a.n_tiles;
    uint32_t tile = blockIdx.x;
    if (tile < n_tiles) ring.issue(0, tile);
    Tally tally(a);
    uint32_t it = 0;
    for (; tile < n_tiles; tile += gridDim.x, ++it) {
        const uint32_t next = tile + gridDim.x;
        if (next < n_tiles) ring.issue((it + 1u) & 1u, next);
        const uint8_t* base = ring.wait(it);

        // this lane's 64 message bytes: 4 x LDS.128, chunk index XOR-swizzled by (row>>1)&3 (CU_TENSOR_MAP_SWIZZLE_64B)
        uint32_t m[16];
        const uint8_t* row = base + ul * 64;
        const int sw = (ul >> 1) & 3;
#pragma unroll
        for (int c = 0; c < 4; ++c) {
            uint4 q = *reinterpret_cast<const uint4*>(row + ((c ^ sw) << 4));
            m[4 * c + 0] = bswap(q.x); m[4 * c + 1] = bswap(q.y); m[4 * c + 2] = bswap(q.z); m[4 * c + 3] = bswap(q.w);   // :34-40
        }
        __syncthreads();                                      // tile drained -> may be refilled next iteration

        const unsigned long long local = (unsigned long long)tile * TU + ul;
        const bool valid = local < a.n_units;
        const unsigned long long gunit = a.unit_base + local;

        uint32_t fs0 = 0xFFFFFFFFu, fs1 = 0xFFFFFFFFu, fmask = 0u;
        if (INJECT) {
            Fault f = fault_for_unit(a, NC, valid ? local : 0ull, [](uint32_t) { return 32u; });
            if (f.active && valid) {
                if (Lanes<NC>::voter(lane)) tally.injected++;
                if ((int)f.replica == r) {
                    fmask = 1u << f.bit;
                    if (f.site < SHA_SITES_PER_BLOCK) fs0 = f.site; else fs1 = f.site - SHA_SITES_PER_BLOCK;
                }
            }
        }

        uint32_t st[8];
        sha_init(st);
        sha_compress<INJECT>(st, m, fs0, fmask);              // :119-127 first (and only) full block
        // :132-163 padding block of a 64-byte message: 0x80, zeros, bit length 512
#pragma unroll
        for (int i = 0; i < 16; ++i) m[i] = 0u;
        m[0] = 0x80000000u; m[15] = 512u;
        sha_compress<INJECT, true>(st, m, fs1, fmask);        // :164

        sha_vote_store<NC>(st, static_cast<uint8_t*>(a.out), local, gunit, valid, lane, a.flags, tally);
    }
    tally.flush(a.counters);
}

// ---------------------------------------------------------------------------------------------
// General path: any unit_bytes (the 10-byte and 4000-byte KATs, ragged sizes).  Bytes are read
// straight from global memory; one thread = one replica of one message; same lane layout/voter.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t sha_padded_byte(const uint8_t* msg, uint32_t len, uint32_t pos) {
    return pos < len ? (uint32_t)__ldg(msg + pos) : (pos == len ? 0x80u : 0u);
}

template <int NC, bool INJECT>
__device__ __forceinline__ void sha256_gen_body(const xmr_args& a) {
    constexpr int UPW = Lanes<NC>::kUnitsPerWarp;
    const int lane = threadIdx.x & 31;
    const int r = Lanes<NC>::replica(lane);
    const unsigned long long gwarp = ((unsigned long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const unsigned long long nwarps = ((unsigned long long)gridDim.x * blockDim.x) >> 5;
    const uint32_t len = a.unit_bytes;
    const uint32_t nblk = (len + 8u) / 64u + 1u;
    const unsigned long long n_wtiles = (a.n_units + UPW - 1) / UPW;
    Tally tally(a);
    for (unsigned long long wt = gwarp; wt < n_wtiles; wt += nwarps) {
        const unsigned long long local = wt * UPW + Lanes<NC>::unit(lane);
        const bool valid = local < a.n_units;
        const unsigned long long gunit = a.unit_base + local;
        const uint8_t* msg = static_cast<const uint8_t*>(a.in) + (valid ? local : 0ull) * len;
        uint32_t fsite = 0xFFFFFFFFu, fmask = 0u;
        if (INJECT) {
            Fault f = fault_for_unit(a, NC, valid ? local : 0ull, [](uint32_t) { return 32u; });
            if (f.active && valid) {
                if (Lanes<NC>::voter(lane)) tally.injected++;
                if ((int)f.replica == r) { fmask = 1u << f.bit; fsite = f.site; }
            }
        }
        const bool sv = (a.flags & XMR_F_STORE_VOTES) != 0;
        const bool majority = a.flags & COAST_F_MAJORITY_VOTER;
        uint32_t sv_bad = 0;
        uint32_t st[8];
        sha_init(st);
        // r02: whole blocks come in as 4 x 16-byte (or 16 x 4-byte) loads when every message is that aligned; the byte walk
        // is left for the padded tail and for unaligned batches (r01 fetched 64 single bytes per block)
        const uintptr_t al = reinterpret_cast<uintptr_t>(a.in) | len;
        for (uint32_t blk = 0; blk < nblk; ++blk) {
            uint32_t m[16];
            if ((al & 15u) == 0 && blk * 64u + 64u <= len) {
#pragma unroll
                for (int c = 0; c < 4; ++c) {
                    const uint4 q = __ldg(reinterpret_cast<const uint4*>(msg + blk * 64u) + c);
                    m[4 * c + 0] = bswap(q.x); m[4 * c + 1] = bswap(q.y); m[4 * c + 2] = bswap(q.z); m[4 * c + 3] = bswap(q.w);
                }
            } else {
#pragma unroll
                for (int w = 0; w < 16; ++w) {
                    const uint32_t p = blk * 64u + 4u * w;
                    if ((al & 3u) == 0 && p + 4u <= len) m[w] = bswap(__ldg(reinterpret_cast<const uint32_t*>(msg + p)));
                    else m[w] = (sha_padded_byte(msg, len, p) << 24) | (sha_padded_byte(msg, len, p + 1) << 16) |
                                (sha_padded_byte(msg, len, p + 2) << 8) | sha_padded_byte(msg, len, p + 3);
                }
            }
            if (blk == nblk - 1) {                            // :155-163, 64-bit big-endian bit count
                m[14] = len >> 29;
                m[15] = len << 3;
            }
            uint32_t fs = (INJECT && fsite / SHA_SITES_PER_BLOCK == blk) ? fsite % SHA_SITES_PER_BLOCK : 0xFFFFFFFFu;
            if (!sv) {
                sha_compress<INJECT>(st, m, fs, fmask);
            } else {
                // ctx_data[k] = data[i] (:120): one u8 vote per MESSAGE byte of this block (padding and length bytes are constants /
                // control state), on the big-endian-packed words
                const uint32_t lo = blk * 64u, nmsg = len > lo ? (len - lo < 64u ? len - lo : 64u) : 0u;
#pragma unroll
                for (int w = 0; w < 16; ++w) {
                    const uint32_t nb = nmsg > 4u * w ? (nmsg - 4u * w < 4u ? nmsg - 4u * w : 4u) : 0u;
                    sv_bad += store_vote_bytes<NC>(m[w], nb, lane, majority);
                }
                sv_bad += sha_compress_sv<NC, INJECT>(st, m, fs, fmask, lane, majority);
            }
        }
        if (!sv) {
            sha_vote_store<NC>(st, static_cast<uint8_t*>(a.out), local, gunit, valid, lane, a.flags, tally);
        } else {                                              // the SoR exit with the in-loop disagreements added: len + 720 per compression + 32 votes
            uint32_t o[8], bad = 0;
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

// ---------------------------------------------------------------------------------------------
// TMR, segmented layout (-s, the reference's default replica scheduling, interface.cpp:245-247):
// the three replicas of a unit sit on the SAME lane of three ADJACENT WARPS, so all 32 lanes of every
// warp carry a unit (the interleaved layout idles 2 of 32 lanes).  CTA = 12 warps = 4 groups x 3 replica
// warps; tile = 128 messages through the same TMA ring.  SoR exit: replica warps 1 and 2 publish their
// state through shared memory, a 96-thread named barrier per group orders it, warp 0 of the group votes
// (same select voter / counters) and stores 32 lanes x 32 B = 1 KiB contiguous.
// ---------------------------------------------------------------------------------------------
constexpr int SEG_THREADS = XMR_SHA_SEG_THREADS, SEG_GROUPS = SEG_THREADS / 96, SEG_TU = SEG_GROUPS * 32;
constexpr uint32_t SEG_EXCH_WORDS = 2 * 8 * 32;              // per tile parity and group: [replica 1..2][word][lane]

template <bool INJECT>
__device__ __forceinline__ void sha256_b64_seg_body(const xmr_args& a, const CUtensorMap* tmap) {
    using Ring = TileRing<SEG_TU, 64>;
    static_assert(SEG_TU == XMR_SHA_SEG_TILE_ROWS && Ring::SMEM_BYTES <= xmr_sha_seg_exch_offset() &&
                  xmr_sha_seg_exch_offset() + 2u * SEG_GROUPS * SEG_EXCH_WORDS * 4u <= xmr_sha_seg_smem(),
                  "ring and exchange buffer fit the launch's shared memory");
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    Ring ring;
    ring.init(smem_raw, tmap);
    // exchange buffer [parity][group][replica 1..2][word][lane]
    uint32_t* exch = reinterpret_cast<uint32_t*>(smem_raw + xmr_sha_seg_exch_offset());
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int g = warp / 3, r = warp - 3 * g;
    const int ul = g * 32 + lane;
    const uint32_t n_tiles = a.n_tiles;
    const bool majority = a.flags & COAST_F_MAJORITY_VOTER;
    uint32_t tile = blockIdx.x;
    if (tile < n_tiles) ring.issue(0, tile);
    Tally tally(a);
    uint32_t it = 0;
    for (; tile < n_tiles; tile += gridDim.x, ++it) {
        const uint32_t next = tile + gridDim.x;
        if (next < n_tiles) ring.issue((it + 1u) & 1u, next);
        const uint8_t* base = ring.wait(it);
        uint32_t m[16];
        const uint8_t* row = base + ul * 64;
        const int sw = (ul >> 1) & 3;
#pragma unroll
        for (int c = 0; c < 4; ++c) {
            uint4 q = *reinterpret_cast<const uint4*>(row + ((c ^ sw) << 4));
            m[4 * c + 0] = bswap(q.x); m[4 * c + 1] = bswap(q.y); m[4 * c + 2] = bswap(q.z); m[4 * c + 3] = bswap(q.w);
        }
        __syncthreads();
        const unsigned long long local = (unsigned long long)tile * SEG_TU + ul;
        const bool valid = local < a.n_units;
        uint32_t fs0 = 0xFFFFFFFFu, fs1 = 0xFFFFFFFFu, fmask = 0u;
        if (INJECT) {
            Fault f = fault_for_unit(a, 3, valid ? local : 0ull, [](uint32_t) { return 32u; });
            if (f.active && valid) {
                if (r == 0) tally.injected++;
                if ((int)f.replica == r) {
                    fmask = 1u << f.bit;
                    if (f.site < SHA_SITES_PER_BLOCK) fs0 = f.site; else fs1 = f.site - SHA_SITES_PER_BLOCK;
                }
            }
        }
        uint32_t st[8];
        sha_init(st);
        sha_compress<INJECT>(st, m, fs0, fmask);
#pragma unroll
        for (int i = 0; i < 16; ++i) m[i] = 0u;
        m[0] = 0x80000000u; m[15] = 512u;
        sha_compress<INJECT, true>(st, m, fs1, fmask);

        uint32_t* ex = exch + ((it & 1u) * SEG_GROUPS + g) * SEG_EXCH_WORDS;
        if (r > 0) {
#pragma unroll
            for (int i = 0; i < 8; ++i) ex[((r - 1) * 8 + i) * 32 + lane] = st[i];
        }
        // the group's 3 warps (96 threads); ids are immediates so only 5 hardware barriers are reserved (0 = __syncthreads)
        if (g == 0) asm volatile("bar.sync 1, 96;" ::: "memory");
        else if (g == 1) asm volatile("bar.sync 2, 96;" ::: "memory");
        else if (g == 2) asm volatile("bar.sync 3, 96;" ::: "memory");
        else asm volatile("bar.sync 4, 96;" ::: "memory");
        if (r == 0) {
            uint32_t o[8], bad = 0;
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                const uint32_t x = st[i], r1 = ex[i * 32 + lane], r2 = ex[(8 + i) * 32 + lane];
                const uint32_t e01 = __vcmpeq4(x, r1), e02 = __vcmpeq4(x, r2);
                const uint32_t v = majority ? ((x & r1) | (x & r2) | (r1 & r2)) : ((x & e01) | (r2 & ~e01));
                bad += __popc(~(e01 & e02)) >> 3;
                o[i] = bswap(v);
            }
            if (valid) {
                uint4* dst = reinterpret_cast<uint4*>(static_cast<uint8_t*>(a.out) + local * 32ull);
                dst[0] = make_uint4(o[0], o[1], o[2], o[3]);
                dst[1] = make_uint4(o[4], o[5], o[6], o[7]);
                tally.unit_exit<3>(bad, 32u, a.flags, a.unit_base + local);
            }
        }
        // exch is double-buffered by tile parity; the __syncthreads of the next iteration orders its reuse
    }
    tally.flush(a.counters);
}

}  // namespace xmr

#define XMR_SHA_B64_KERNEL(NC, INJ)                                                                      \
    extern "C" __global__ void __launch_bounds__(XMR_CTA_THREADS)                                        \
    xmr_sha256_b64_nc##NC##_inj##INJ(const __grid_constant__ xmr_args a, const __grid_constant__ CUtensorMap tmap) { \
        xmr::sha256_b64_body<NC, INJ != 0>(a, &tmap);                                                    \
    }
#define XMR_SHA_GEN_KERNEL(NC, INJ)                                                                      \
    extern "C" __global__ void __launch_bounds__(XMR_CTA_THREADS)                                        \
    xmr_sha256_gen_nc##NC##_inj##INJ(const __grid_constant__ xmr_args a) {                               \
        xmr::sha256_gen_body<NC, INJ != 0>(a);                                                           \
    }
XMR_SHA_B64_KERNEL(1, 0) XMR_SHA_B64_KERNEL(2, 0) XMR_SHA_B64_KERNEL(3, 0)
XMR_SHA_B64_KERNEL(1, 1) XMR_SHA_B64_KERNEL(2, 1) XMR_SHA_B64_KERNEL(3, 1)
XMR_SHA_GEN_KERNEL(1, 0) XMR_SHA_GEN_KERNEL(2, 0) XMR_SHA_GEN_KERNEL(3, 0)
XMR_SHA_GEN_KERNEL(1, 1) XMR_SHA_GEN_KERNEL(2, 1) XMR_SHA_GEN_KERNEL(3, 1)

#define XMR_SHA_B64_SEG_KERNEL(INJ)                                                                      \
    extern "C" __global__ void __launch_bounds__(xmr::SEG_THREADS)                                       \
    xmr_sha256_b64_seg_nc3_inj##INJ(const __grid_constant__ xmr_args a, const __grid_constant__ CUtensorMap tmap) { \
        xmr::sha256_b64_seg_body<INJ != 0>(a, &tmap);                                                    \
    }
XMR_SHA_B64_SEG_KERNEL(0) XMR_SHA_B64_SEG_KERNEL(1)
