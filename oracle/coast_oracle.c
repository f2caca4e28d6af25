/*
 * coast_oracle.c -- CPU oracle (TEST INFRASTRUCTURE ONLY; see coast_oracle.h).
 *
 * Every function cites the reference file:line it restates.  Paths are relative
 * to the byuccl/coast checkout (commit 397a26e).
 */
#include "coast_oracle.h"

#include <pthread.h>
#include <stdlib.h>
#include <string.h>

/* ------------------------------------------------------------------ */
/* Philox4x32-10                                                        */
/* ------------------------------------------------------------------ */
void orc_philox4x32_10(const uint32_t ctr[4], const uint32_t key[2], uint32_t out[4]) {
    uint32_t c0 = ctr[0], c1 = ctr[1], c2 = ctr[2], c3 = ctr[3];
    uint32_t k0 = key[0], k1 = key[1];
    for (int r = 0; r < 10; ++r) {
        uint64_t p0 = (uint64_t)0xD2511F53u * c0;
        uint64_t p1 = (uint64_t)0xCD9E8D57u * c2;
        uint32_t n0 = (uint32_t)(p1 >> 32) ^ c1 ^ k0;
        uint32_t n1 = (uint32_t)p1;
        uint32_t n2 = (uint32_t)(p0 >> 32) ^ c3 ^ k1;
        uint32_t n3 = (uint32_t)p0;
        c0 = n0; c1 = n1; c2 = n2; c3 = n3;
        k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
    }
    out[0] = c0; out[1] = c1; out[2] = c2; out[3] = c3;
}

void orc_fill_philox(uint32_t* dst, uint64_t n_words, uint64_t word_base, uint32_t seed) {
    uint32_t key[2] = { seed, 0 };
    uint32_t ctr[4] = { 0, 0, 0, 0 }, x[4];
    uint64_t cur = ~(uint64_t)0;
    for (uint64_t i = 0; i < n_words; ++i) {
        uint64_t w = word_base + i, blk = w >> 2;
        if (blk != cur) {
            ctr[0] = (uint32_t)blk; ctr[1] = (uint32_t)(blk >> 32);
            orc_philox4x32_10(ctr, key, x);
            cur = blk;
        }
        dst[i] = x[w & 3];
    }
}

/* ------------------------------------------------------------------ */
/* Fault-site geometry and the per-unit fault decision                  */
/* (fault model: simulation/platform/resources/injector.py:202-207 --   */
/*  one single-bit flip `val ^ (1 << bit)` per run; a run = one unit)   */
/* ------------------------------------------------------------------ */
#define SHA_SITES_PER_BLOCK 536u /* 16 m[] + 64*8 working vars + 8 ctx_state */
#define CHS_SITES_PER_BLOCK 421u /* CHStone sha: 16 W[] + 80*5 working vars + 5 sha_info_digest */

static uint32_t sha_blocks(uint32_t len) { return (len + 8u) / 64u + 1u; }

uint32_t orc_fault_sites(uint32_t kernel, uint32_t unit_bytes, uint32_t K) {
    switch (kernel) {
    case ORC_K_CHSTONE_AES: return 176u;
    case ORC_K_CRC16:     return 2u * unit_bytes;
    case ORC_K_SHA256:    return SHA_SITES_PER_BLOCK * sha_blocks(unit_bytes);
    case ORC_K_AES128:    return 16u + 160u;
    case ORC_K_MM_U32:    return K;
    case ORC_K_GEMM_TF32: return 1u;
    case ORC_K_QSORT:     return 33u * (unit_bytes / 4u);   /* 32*L dynamic compare events + L input-copy elements */
    case ORC_K_CHSTONE_SHA: return CHS_SITES_PER_BLOCK * (unit_bytes / 64u + 1u);
    default:              return 0u;
    }
}

uint32_t orc_fault_site_bits(uint32_t kernel, uint32_t unit_bytes, uint32_t K, uint32_t site) {
    (void)K;
    switch (kernel) {
    case ORC_K_CRC16:  return site < unit_bytes ? 16u : 8u;
    case ORC_K_AES128: return 8u;
    case ORC_K_CHSTONE_AES: return 8u;         /* statemt[] holds one byte per int (aes.c:83); above bit 7 the S-box index leaves the table */
    default:           return 32u;
    }
}

uint32_t orc_out_bytes_per_unit(uint32_t kernel) {
    switch (kernel) {
    case ORC_K_CRC16: return 2; case ORC_K_SHA256: return 32; case ORC_K_AES128: return 16;
    case ORC_K_MM_U32: case ORC_K_GEMM_TF32: return 4; case ORC_K_CHSTONE_SHA: return 20; case ORC_K_CHSTONE_AES: return 64; default: return 0;
    }
}

/* One vote per output element OF THE C TYPE THE REFERENCE STORES (SURVEY.md 7):
 * u16 crc (crc16.c:30), u8 digest byte (sha256_common_tmr.c:169-178),
 * u8 state byte (TI_aes_128.c:226-229), mm_t element (mm_common_tmr.c:16),
 * LONG sha_info_digest word (chstone/sha/sha.h:38, compared in sha_driver.c:59). */
uint32_t orc_out_bytes(uint32_t kernel, uint32_t unit_bytes) {
    return kernel == ORC_K_QSORT ? unit_bytes : orc_out_bytes_per_unit(kernel);
}

uint32_t orc_votes_per_unit(uint32_t kernel) {
    switch (kernel) {
    case ORC_K_CRC16: return 1; case ORC_K_SHA256: return 32; case ORC_K_AES128: return 16;
    case ORC_K_MM_U32: case ORC_K_GEMM_TF32: return 1; case ORC_K_CHSTONE_SHA: return 5;
    case ORC_K_CHSTONE_AES: return 16;                      /* int statemt[i], compared element-wise (aes_enc.c:130-131) */
    default: return 0;
    }
}

void orc_fault_for_unit(const orc_plan* plan, uint32_t kernel, uint32_t num_clones, uint32_t unit_bytes,
                        uint32_t K, uint64_t unit, uint64_t local, orc_fault* f) {
    f->active = 0; f->replica = f->site = f->bit = 0;
    if (!plan || plan->mode == ORC_PLAN_NONE) return;
    uint32_t ns = orc_fault_sites(kernel, unit_bytes, K);
    if (ns == 0) return;
    if (plan->mode == ORC_PLAN_BERNOULLI) {
        uint32_t ctr[4] = { (uint32_t)unit, (uint32_t)(unit >> 32), 0, 0 };
        uint32_t key[2] = { plan->seed_lo, plan->seed_hi }, x[4];
        orc_philox4x32_10(ctr, key, x);
        if (x[0] >= plan->threshold) return;
        f->replica = x[1] % num_clones;
        f->site = x[2] % ns;
        f->bit = x[3] % orc_fault_site_bits(kernel, unit_bytes, K, f->site);
        f->active = 1;
    } else if (plan->mode == ORC_PLAN_TABLE && plan->table) {
        uint32_t e = plan->table[local];
        if (!(e & 0x80000000u)) return;
        uint32_t rep = (e >> 29) & 3u, site = (e >> 5) & 0xFFFFFFu, bit = e & 31u;
        if (rep >= num_clones || site >= ns) return;
        if (bit >= orc_fault_site_bits(kernel, unit_bytes, K, site)) return;
        f->replica = rep; f->site = site; f->bit = bit; f->active = 1;
    }
}

/* ------------------------------------------------------------------ */
/* a1: crc16()  tests/crc16/crc16.c:21-31                               */
/* ------------------------------------------------------------------ */
uint16_t orc_crc16(const uint8_t* data, uint32_t len, const orc_fault* f) {
    uint16_t crc = 0xFFFF;                                  /* crc16.c:23 */
    for (uint32_t n = 0; n < len; ++n) {                    /* crc16.c:25 while (length--) */
        uint8_t b = data[n];
        if (f && f->active && f->site == len + n) b ^= (uint8_t)(1u << f->bit);
        uint8_t x = (uint8_t)((crc >> 8) ^ b);              /* :26 (u8 truncation) */
        x ^= (uint8_t)(x >> 4);                             /* :27 */
        crc = (uint16_t)((uint16_t)(crc << 8) ^ (uint16_t)((uint16_t)x << 12) ^
                         (uint16_t)((uint16_t)x << 5) ^ (uint16_t)x); /* :28 */
        if (f && f->active && f->site == n) crc ^= (uint16_t)(1u << f->bit);
    }
    return crc;                                             /* :30, the voted `ret i16` */
}

/* ------------------------------------------------------------------ */
/* a2/a3: sha256_transform / sha256_hash                                 */
/*        tests/sha256_common/sha256_common_tmr.c:28-98, 101-180         */
/* ------------------------------------------------------------------ */
static const uint32_t SHA_K[64] = { /* FIPS 180-4 4.2.2; same values as sha256_common_tmr.c:8-19 */
    0x428a2f98u, 0x71374491u, 0xb5c0fbcfu, 0xe9b5dba5u, 0x3956c25bu, 0x59f111f1u, 0x923f82a4u, 0xab1c5ed5u,
    0xd807aa98u, 0x12835b01u, 0x243185beu, 0x550c7dc3u, 0x72be5d74u, 0x80deb1feu, 0x9bdc06a7u, 0xc19bf174u,
    0xe49b69c1u, 0xefbe4786u, 0x0fc19dc6u, 0x240ca1ccu, 0x2de92c6fu, 0x4a7484aau, 0x5cb0a9dcu, 0x76f988dau,
    0x983e5152u, 0xa831c66du, 0xb00327c8u, 0xbf597fc7u, 0xc6e00bf3u, 0xd5a79147u, 0x06ca6351u, 0x14292967u,
    0x27b70a85u, 0x2e1b2138u, 0x4d2c6dfcu, 0x53380d13u, 0x650a7354u, 0x766a0abbu, 0x81c2c92eu, 0x92722c85u,
    0xa2bfe8a1u, 0xa81a664bu, 0xc24b8b70u, 0xc76c51a3u, 0xd192e819u, 0xd6990624u, 0xf40e3585u, 0x106aa070u,
    0x19a4c116u, 0x1e376c08u, 0x2748774cu, 0x34b0bcb5u, 0x391c0cb3u, 0x4ed8aa4au, 0x5b9cca4fu, 0x682e6ff3u,
    0x748f82eeu, 0x78a5636fu, 0x84c87814u, 0x8cc70208u, 0x90befffau, 0xa4506cebu, 0xbef9a3f7u, 0xc67178f2u };

static inline uint32_t rotr32(uint32_t v, unsigned n) { return (v >> n) | (v << (32u - n)); }

/* One compression; `blk` = index of this compression in the message (fault sites are
 * numbered blk*536 + s). */
static void sha_compress(uint32_t st[8], const uint8_t blk_bytes[64], uint32_t blk, const orc_fault* f) {
    uint32_t m[64], v[8];
    int has = f && f->active && (f->site / SHA_SITES_PER_BLOCK) == blk;
    uint32_t s = has ? f->site % SHA_SITES_PER_BLOCK : 0xFFFFFFFFu;
    uint32_t mask = has ? (1u << f->bit) : 0u;
    for (int i = 0; i < 16; ++i)                            /* :34-40 big-endian pack */
        m[i] = ((uint32_t)blk_bytes[4 * i] << 24) | ((uint32_t)blk_bytes[4 * i + 1] << 16) |
               ((uint32_t)blk_bytes[4 * i + 2] << 8) | (uint32_t)blk_bytes[4 * i + 3];
    if (s < 16u) m[s] ^= mask;
    for (int i = 16; i < 64; ++i) {                         /* :42-58 */
        uint32_t a = m[i - 2], b = m[i - 15];
        uint32_t s1 = rotr32(a, 17) ^ rotr32(a, 19) ^ (a >> 10);
        uint32_t s0 = rotr32(b, 7) ^ rotr32(b, 18) ^ (b >> 3);
        m[i] = s1 + m[i - 7] + s0 + m[i - 16];
    }
    for (int i = 0; i < 8; ++i) v[i] = st[i];               /* :60-67 */
    for (uint32_t t = 0; t < 64; ++t) {                     /* :69-88 */
        if (s >= 16u && s < 528u && (s - 16u) / 8u == t) v[(s - 16u) % 8u] ^= mask;
        uint32_t a = v[0], b = v[1], c = v[2], e = v[4], ff = v[5], g = v[6];
        uint32_t ep0 = rotr32(a, 2) ^ rotr32(a, 13) ^ rotr32(a, 22);
        uint32_t ep1 = rotr32(e, 6) ^ rotr32(e, 11) ^ rotr32(e, 25);
        uint32_t ch = (e & ff) ^ (~e & g);
        uint32_t maj = (a & b) ^ (a & c) ^ (b & c);
        uint32_t t1 = v[7] + ep1 + ch + SHA_K[t] + m[t];
        uint32_t t2 = ep0 + maj;
        v[7] = g; v[6] = ff; v[5] = e; v[4] = v[3] + t1; v[3] = c; v[2] = b; v[1] = a; v[0] = t1 + t2;
    }
    for (int i = 0; i < 8; ++i) st[i] += v[i];              /* :90-97 */
    if (s >= 528u && s < 536u) st[s - 528u] ^= mask;
}

void orc_sha256(const uint8_t* data, uint32_t len, uint8_t digest[32], const orc_fault* f) {
    uint32_t st[8] = { 0x6a09e667u, 0xbb67ae85u, 0x3c6ef372u, 0xa54ff53au,   /* :108-115 */
                       0x510e527fu, 0x9b05688cu, 0x1f83d9abu, 0x5be0cd19u };
    uint8_t buf[64];
    uint32_t blk = 0, off = 0;
    while (len - off >= 64u) {                              /* :119-127 (byte feed, transform each 64) */
        sha_compress(st, data + off, blk++, f);
        off += 64u;
    }
    uint32_t rem = len - off;                               /* ctx_datalen */
    memcpy(buf, data + off, rem);
    buf[rem] = 0x80;                                        /* :133 / :137 */
    if (rem < 56u) {
        memset(buf + rem + 1, 0, 55u - rem);                /* :134-135 */
    } else {
        memset(buf + rem + 1, 0, 63u - rem);                /* :138-139 */
        sha_compress(st, buf, blk++, f);                    /* :140 */
        memset(buf, 0, 56);                                 /* :142-151 */
    }
    /* :155-163: bitlen = 512*full_blocks + 8*rem as a 64-bit big-endian count
     * (DBL_INT_ADD carries bitlen[0] overflow into bitlen[1]). */
    uint64_t bits = (uint64_t)len * 8u;
    for (int i = 0; i < 8; ++i) buf[63 - i] = (uint8_t)(bits >> (8 * i));
    sha_compress(st, buf, blk++, f);                        /* :164 */
    for (int w = 0; w < 8; ++w)                             /* :169-178 big-endian digest bytes */
        for (int i = 0; i < 4; ++i) digest[4 * w + i] = (uint8_t)(st[w] >> (24 - 8 * i));
}

/* ------------------------------------------------------------------ */
/* 8f-4: CHStone sha  tests/chstone/sha/sha.c                            */
/* The CHStone variant: no rotate in the W expansion (USE_MODIFIED_SHA is */
/* not defined, :101), LITTLE-endian word load (its own memcpy, :71-90),  */
/* and a final block indexed in WORDS by a BYTE count (:167-168).         */
/* A unit is one stream of `len` bytes, len a multiple of 64 below 2^29:  */
/* sha_init; sha_update over whole 64-byte blocks (:149-154; the trailing */
/* memcpy :155 copies nothing); sha_final with count == 0, i.e.           */
/* data[0] = 0x80 (:168), data[1..13] = 0 (its own memset, :174 -> :55-69 */
/* zeroes (56-1)/4 = 13 words after skipping 1), data[14] = hi = 0,       */
/* data[15] = lo = 8*len (:176-177).  sha_stream (:182-193) over chunks   */
/* in_i[j] that are multiples of 64 is the same thing on the concatenation*/
/* ------------------------------------------------------------------ */
static inline uint32_t rotl32(uint32_t v, unsigned n) { return (v << n) | (v >> (32u - n)); }

static void chs_transform(uint32_t dig[5], const uint32_t data[16], uint32_t blk, const orc_fault* f) {
    uint32_t W[80], v[5];
    int has = f && f->active && (f->site / CHS_SITES_PER_BLOCK) == blk;
    uint32_t s = has ? f->site % CHS_SITES_PER_BLOCK : 0xFFFFFFFFu;
    uint32_t mask = has ? (1u << f->bit) : 0u;
    for (int i = 0; i < 16; ++i) W[i] = data[i];                               /* :97-99 */
    if (s < 16u) W[s] ^= mask;
    for (int i = 16; i < 80; ++i) W[i] = W[i - 3] ^ W[i - 8] ^ W[i - 14] ^ W[i - 16];   /* :100-102 */
    for (int i = 0; i < 5; ++i) v[i] = dig[i];                                 /* :103-107 */
    for (uint32_t t = 0; t < 80; ++t) {                                        /* :109-120, FUNC :47-53 */
        if (s >= 16u && s < 416u && (s - 16u) / 5u == t) v[(s - 16u) % 5u] ^= mask;
        uint32_t A = v[0], B = v[1], C = v[2], D = v[3], E = v[4], fn, k;
        if (t < 20)      { fn = (B & C) | (~B & D);          k = 0x5a827999u; }   /* f1 :30 */
        else if (t < 40) { fn = B ^ C ^ D;                   k = 0x6ed9eba1u; }   /* f2 :31 */
        else if (t < 60) { fn = (B & C) | (B & D) | (C & D); k = 0x8f1bbcdcu; }   /* f3 :32 */
        else             { fn = B ^ C ^ D;                   k = 0xca62c1d6u; }   /* f4 :33 */
        uint32_t temp = rotl32(A, 5) + fn + E + W[t] + k;
        v[4] = D; v[3] = C; v[2] = rotl32(B, 30); v[1] = A; v[0] = temp;
    }
    for (int i = 0; i < 5; ++i) dig[i] += v[i];                                /* :122-126 */
    if (s >= 416u && s < 421u) dig[s - 416u] ^= mask;
}

void orc_chstone_sha(const uint8_t* data, uint32_t len, uint32_t digest[5], const orc_fault* f) {
    uint32_t dig[5] = { 0x67452301u, 0xefcdab89u, 0x98badcfeu, 0x10325476u, 0xc3d2e1f0u };   /* :132-136 */
    uint32_t w[16], blk = 0;
    for (uint32_t off = 0; off + 64u <= len; off += 64u) {                     /* :149-154 */
        for (int i = 0; i < 16; ++i)                                           /* :78-89 little-endian pack */
            w[i] = (uint32_t)data[off + 4 * i] | ((uint32_t)data[off + 4 * i + 1] << 8) |
                   ((uint32_t)data[off + 4 * i + 2] << 16) | ((uint32_t)data[off + 4 * i + 3] << 24);
        chs_transform(dig, w, blk++, f);
    }
    memset(w, 0, sizeof w);
    w[0] = 0x80u; w[14] = 0u; w[15] = len << 3;                                /* :168, :174, :176-177 */
    chs_transform(dig, w, blk, f);                                             /* :178 */
    for (int i = 0; i < 5; ++i) digest[i] = dig[i];
}

/* ------------------------------------------------------------------ */
/* a5: aes_enc_dec()  tests/aes/TI_aes_128.c:107-231                     */
/* Tables are GENERATED (FIPS-197 5.1.1: GF(2^8) inverse + affine map)   */
/* rather than transcribed; they equal TI_aes_128.c:44-61,64-80,83-84.   */
/* ------------------------------------------------------------------ */
static uint8_t AES_S[256], AES_IS[256], AES_RC[10];
static pthread_once_t aes_once = PTHREAD_ONCE_INIT;

static uint8_t gf_xtime(uint8_t v) { return (uint8_t)((v << 1) ^ ((v & 0x80) ? 0x1b : 0)); } /* galois_mul2 :88-99 */
static uint8_t gf_mul(uint8_t a, uint8_t b) {
    uint8_t p = 0;
    while (b) { if (b & 1) p ^= a; a = gf_xtime(a); b >>= 1; }
    return p;
}
static void aes_tables(void) {
    for (int x = 0; x < 256; ++x) {
        uint8_t inv = 0;
        if (x) for (int y = 1; y < 256; ++y) if (gf_mul((uint8_t)x, (uint8_t)y) == 1) { inv = (uint8_t)y; break; }
        uint8_t s = inv, r = inv;
        for (int i = 0; i < 4; ++i) { r = (uint8_t)((r << 1) | (r >> 7)); s ^= r; }
        s ^= 0x63;
        AES_S[x] = s; AES_IS[s] = (uint8_t)x;
    }
    uint8_t rc = 1;
    for (int i = 0; i < 10; ++i) { AES_RC[i] = rc; rc = gf_xtime(rc); }
}

static void aes_key_fwd(uint8_t k[16], int round) {          /* :214-221 and :114-122 */
    k[0] ^= AES_S[k[13]] ^ AES_RC[round];
    k[1] ^= AES_S[k[14]];
    k[2] ^= AES_S[k[15]];
    k[3] ^= AES_S[k[12]];
    for (int i = 4; i < 16; ++i) k[i] ^= k[i - 4];
}
static void aes_key_bwd(uint8_t k[16], int round) {          /* :134-141; `round` is the Rcon index */
    for (int i = 15; i > 3; --i) k[i] ^= k[i - 4];
    k[0] ^= AES_S[k[13]] ^ AES_RC[round];
    k[1] ^= AES_S[k[14]];
    k[2] ^= AES_S[k[15]];
    k[3] ^= AES_S[k[12]];
}
static void aes_shift_rows(uint8_t s[16], int inverse) {     /* :147-166 / :187-206; state[4*col+row] */
    uint8_t t[16];
    for (int c = 0; c < 4; ++c)
        for (int r = 0; r < 4; ++r) {
            int src = inverse ? ((c - r) & 3) : ((c + r) & 3);
            t[4 * c + r] = s[4 * src + r];
        }
    memcpy(s, t, 16);
}
static void aes_mix_columns(uint8_t s[16], int inverse) {    /* :169-184 (TI's inverse = pre-multiply trick :173-177) */
    for (int c = 0; c < 4; ++c) {
        uint8_t* p = s + 4 * c;
        uint8_t a0 = p[0], a1 = p[1], a2 = p[2], a3 = p[3];
        if (!inverse) {
            p[0] = (uint8_t)(gf_mul(a0, 2) ^ gf_mul(a1, 3) ^ a2 ^ a3);
            p[1] = (uint8_t)(a0 ^ gf_mul(a1, 2) ^ gf_mul(a2, 3) ^ a3);
            p[2] = (uint8_t)(a0 ^ a1 ^ gf_mul(a2, 2) ^ gf_mul(a3, 3));
            p[3] = (uint8_t)(gf_mul(a0, 3) ^ a1 ^ a2 ^ gf_mul(a3, 2));
        } else {
            p[0] = (uint8_t)(gf_mul(a0, 14) ^ gf_mul(a1, 11) ^ gf_mul(a2, 13) ^ gf_mul(a3, 9));
            p[1] = (uint8_t)(gf_mul(a0, 9) ^ gf_mul(a1, 14) ^ gf_mul(a2, 11) ^ gf_mul(a3, 13));
            p[2] = (uint8_t)(gf_mul(a0, 13) ^ gf_mul(a1, 9) ^ gf_mul(a2, 14) ^ gf_mul(a3, 11));
            p[3] = (uint8_t)(gf_mul(a0, 11) ^ gf_mul(a1, 13) ^ gf_mul(a2, 9) ^ gf_mul(a3, 14));
        }
    }
}

void orc_aes128(uint8_t s[16], uint8_t key[16], int dir, const orc_fault* f) {
    pthread_once(&aes_once, aes_tables);
    int has = f && f->active;
    uint8_t mask = has ? (uint8_t)(1u << f->bit) : 0;
    if (has && f->site < 16u) s[f->site] ^= mask;            /* the replica's private copy of the input */
    if (dir) {
        for (int r = 0; r < 10; ++r) aes_key_fwd(key, r);    /* :112-123 reach the last round key */
        for (int i = 0; i < 16; ++i) s[i] ^= key[i];         /* :126-128 */
    }
    for (int r = 0; r < 10; ++r) {                           /* :132 main loop */
        if (dir) {
            aes_key_bwd(key, 9 - r);                         /* :133-141 */
            if (r > 0) aes_mix_columns(s, 1);                /* :169-184 with dir */
            aes_shift_rows(s, 1);                            /* :187-206 */
            for (int i = 0; i < 16; ++i) s[i] = (uint8_t)(AES_IS[s[i]] ^ key[i]); /* :208-211 */
        } else {
            for (int i = 0; i < 16; ++i) s[i] = AES_S[s[i] ^ key[i]];             /* :143-146 */
            aes_shift_rows(s, 0);                            /* :147-166 */
            if (r < 9) aes_mix_columns(s, 0);                /* :169-184 */
            aes_key_fwd(key, r);                             /* :214-221 */
        }
        if (has && f->site >= 16u && (f->site - 16u) / 16u == (uint32_t)r) s[(f->site - 16u) % 16u] ^= mask;
    }
    if (!dir) for (int i = 0; i < 16; ++i) s[i] ^= key[i];   /* :224-229 */
}

/* ------------------------------------------------------------------ */
/* SURVEY 8f-4: CHStone `aes`  tests/chstone/aes/{aes_enc,aes_dec,aes_func,aes_key}.c, type 128128               */
/* One byte per `int`; the key schedule is expanded once into word[4][44] (KeySchedule aes_key.c:79-165) and the */
/* key itself is never modified.  encrypt() aes_enc.c:66-134: AddRoundKey(0); 9 x {ByteSub_ShiftRow;            */
/* MixColumn_AddRoundKey(i)}; ByteSub_ShiftRow; AddRoundKey(10).  decrypt() aes_dec.c:66-140: AddRoundKey(10);   */
/* InversShiftRow_ByteSub; 9 x {AddRoundKey_InversMixColumn(i); InversShiftRow_ByteSub} for i = 9..1;            */
/* AddRoundKey(0).  The printf and the `main_result +=` self-check inside both functions are host effects of the */
/* benchmark, not part of the protected arithmetic.                                                              */
/* Fault sites: 0..15 = statemt[i] as loaded; 16+16r+i = statemt[i] right after the (r+2)-th round-key addition   */
/* (encrypt: after MixColumn_AddRoundKey(r+1) / the final AddRoundKey; decrypt: after the first loop of          */
/* AddRoundKey_InversMixColumn(9-r) aes_func.c:443-449 / the final AddRoundKey(0)).                              */
/* ------------------------------------------------------------------ */
static int chs_xt(int v) { v <<= 1; if ((v >> 8) == 1) v ^= 283; return v; }           /* the `x << 1; if ((x >> 8) == 1) x ^= 283` idiom */
static void chs_key_schedule(const int32_t key[16], int word[4][44]) {                 /* aes_key.c:129-163, nk = nb = 4, 10 rounds */
    static const int rcon0[10] = { 0x01, 0x02, 0x04, 0x08, 0x10, 0x20, 0x40, 0x80, 0x1b, 0x36 };   /* :64-73 */
    for (int j = 0; j < 4; ++j) for (int i = 0; i < 4; ++i) word[i][j] = key[i + j * 4];
    for (int j = 4; j < 44; ++j) {
        int temp[4];
        if (j % 4 == 0) {                                                               /* RotByte + SubByte :137-143 */
            temp[0] = AES_S[word[1][j - 1] & 0xFF] ^ rcon0[j / 4 - 1];
            temp[1] = AES_S[word[2][j - 1] & 0xFF]; temp[2] = AES_S[word[3][j - 1] & 0xFF]; temp[3] = AES_S[word[0][j - 1] & 0xFF];
        } else {
            for (int i = 0; i < 4; ++i) temp[i] = word[i][j - 1];
        }
        for (int i = 0; i < 4; ++i) word[i][j] = word[i][j - 4] ^ temp[i];
    }
}
static void chs_add_round_key(int st[16], int word[4][44], int n) {                    /* aes_func.c:537-543 */
    for (int j = 0; j < 4; ++j) for (int i = 0; i < 4; ++i) st[i + j * 4] ^= word[i][j + 4 * n];
}
static void chs_bytesub_shiftrow(int st[16]) {                                         /* aes_func.c:141-165: row r rotates left by r */
    int t[16];
    for (int c = 0; c < 4; ++c) for (int r = 0; r < 4; ++r) t[r + 4 * c] = AES_S[st[r + 4 * ((c + r) & 3)] & 0xFF];
    memcpy(st, t, sizeof t);
}
static void chs_inv_shiftrow_bytesub(int st[16]) {                                     /* aes_func.c:261-285 */
    int t[16];
    for (int c = 0; c < 4; ++c) for (int r = 0; r < 4; ++r) t[r + 4 * c] = AES_IS[st[r + 4 * ((c - r) & 3)] & 0xFF];
    memcpy(st, t, sizeof t);
}
static void chs_mixcolumn(int st[16]) {                                                /* aes_func.c:375-426 without the key */
    for (int j = 0; j < 4; ++j) {
        int a[4], o[4];
        for (int i = 0; i < 4; ++i) a[i] = st[i + j * 4];
        for (int i = 0; i < 4; ++i) o[i] = chs_xt(a[i]) ^ (chs_xt(a[(i + 1) & 3]) ^ a[(i + 1) & 3]) ^ a[(i + 2) & 3] ^ a[(i + 3) & 3];
        for (int i = 0; i < 4; ++i) st[i + j * 4] = o[i];
    }
}
static void chs_inv_mixcolumn(int st[16]) {                                            /* aes_func.c:450-503: (14, 11, 13, 9) */
    for (int j = 0; j < 4; ++j) {
        int a[4], o[4];
        for (int i = 0; i < 4; ++i) a[i] = st[i + j * 4];
        for (int i = 0; i < 4; ++i) {
            const int x0 = a[i], x1 = a[(i + 1) & 3], x2 = a[(i + 2) & 3], x3 = a[(i + 3) & 3];
            const int m14 = chs_xt(chs_xt(chs_xt(x0) ^ x0) ^ x0);                       /* ((2x ^ x) 2 ^ x) 2 */
            const int m11 = chs_xt(chs_xt(chs_xt(x1)) ^ x1) ^ x1;                       /* ((2x) 2 ^ x) 2 ^ x */
            const int m13 = chs_xt(chs_xt(chs_xt(x2) ^ x2)) ^ x2;                       /* ((2x ^ x) 2) 2 ^ x */
            const int m9 = chs_xt(chs_xt(chs_xt(x3))) ^ x3;                             /* 8x ^ x */
            o[i] = m14 ^ m11 ^ m13 ^ m9;
        }
        for (int i = 0; i < 4; ++i) st[i + j * 4] = o[i];
    }
}
void orc_chstone_aes(int32_t statemt[16], const int32_t key[16], int dir, const orc_fault* f) {
    pthread_once(&aes_once, aes_tables);
    int word[4][44], st[16];
    const int has = f && f->active;
    for (int i = 0; i < 16; ++i) st[i] = statemt[i];
    if (has && f->site < 16u) st[f->site] ^= (1 << f->bit);                            /* the replica's private copy of the input */
    chs_key_schedule(key, word);
    if (!dir) {
        chs_add_round_key(st, word, 0);                                                 /* aes_enc.c:118 */
        for (int i = 1; i <= 10; ++i) {
            chs_bytesub_shiftrow(st);                                                   /* :121 / :124 */
            if (i < 10) chs_mixcolumn(st);                                              /* :122 MixColumn_AddRoundKey = MixColumn, */
            chs_add_round_key(st, word, i);                                             /*      then the key (:386-387) / :125 */
            if (has && f->site >= 16u && (f->site - 16u) / 16u == (uint32_t)(i - 1)) st[(f->site - 16u) % 16u] ^= (1 << f->bit);
        }
    } else {
        chs_add_round_key(st, word, 10);                                                /* aes_dec.c:115 */
        chs_inv_shiftrow_bytesub(st);                                                   /* :117 */
        for (int i = 9; i >= 1; --i) {
            chs_add_round_key(st, word, i);                                             /* :121 first loop of AddRoundKey_InversMixColumn */
            if (has && f->site >= 16u && (f->site - 16u) / 16u == (uint32_t)(9 - i)) st[(f->site - 16u) % 16u] ^= (1 << f->bit);
            chs_inv_mixcolumn(st);
            chs_inv_shiftrow_bytesub(st);                                               /* :122 */
        }
        chs_add_round_key(st, word, 0);                                                 /* :125 */
        if (has && f->site >= 16u && (f->site - 16u) / 16u == 9u) st[(f->site - 16u) % 16u] ^= (1 << f->bit);
    }
    for (int i = 0; i < 16; ++i) statemt[i] = st[i];
}

/* ------------------------------------------------------------------ */
/* a7: matrix_multiply()  tests/mm_common/mm_common_tmr.c:3-20,          */
/*     tests/matrixMultiply/matrixMultiply.c:95-112                      */
/* `sum` is an unsigned long truncated to mm_t/unsigned on store (:16 /  */
/* :108): only its low 32 bits are observable, so it is kept mod 2^32.   */
/* ------------------------------------------------------------------ */
uint32_t orc_mm_u32_elem(const uint32_t* A, const uint32_t* B, uint32_t K, uint32_t N, uint32_t i, uint32_t j,
                         const orc_fault* f) {
    uint32_t sum = 0;
    for (uint32_t k = 0; k < K; ++k) {
        sum += A[(size_t)i * K + k] * B[(size_t)k * N + j];
        if (f && f->active && f->site == k) sum ^= (1u << f->bit);
    }
    return sum;
}

/* BASELINE config 4 (fp32 on tensor cores): wgmma tf32 reads the top 19 bits
 * of each fp32 operand; accumulation order inside the tensor core is unspecified, so
 * this is a TOLERANCE oracle (exact products of the truncated operands, summed in
 * double, rounded once). */
static float tf32_trunc(float v) {
    uint32_t b; memcpy(&b, &v, 4); b &= 0xFFFFE000u; memcpy(&v, &b, 4); return v;
}
float orc_gemm_tf32_elem(const float* A, const float* B, uint32_t K, uint32_t N, uint32_t i, uint32_t j,
                         const orc_fault* f) {
    double acc = 0.0;
    for (uint32_t k = 0; k < K; ++k)
        acc += (double)tf32_trunc(A[(size_t)i * K + k]) * (double)tf32_trunc(B[(size_t)k * N + j]);
    float r = (float)acc;
    if (f && f->active && f->site == 0) { uint32_t b; memcpy(&b, &r, 4); b ^= (1u << f->bit); memcpy(&r, &b, 4); }
    return r;
}

/* ------------------------------------------------------------------ */
/* SURVEY 8f-4: quick_sort()  tests/quicksort/quicksort.c:121-136         */
/* The one workload whose BRANCHES depend on data, so the sync points are */
/* the conditional-branch conditions inside the loops (populateSyncPoints */
/* synchronization.cpp:146-155, syncTerminator :741-1113, voter :934-938):*/
/* the replicas run in lockstep, every data-dependent condition is voted  */
/* and the ONE control flow follows the voted value; each replica keeps   */
/* swapping inside its own copy of the array (memory replication).  The   */
/* SoR exit votes each stored element.  Recursion is an explicit stack in */
/* the reference's order (left part first, :134-135).                     */
/* Fault sites: s < 32L: the value loaded for the s-th executed data      */
/* comparison (a register flip); 32L <= s < 33L: element s-32L of the     */
/* replica's private copy before sorting (an input-copy flip).            */
/* ------------------------------------------------------------------ */
typedef struct { int nc, majority, count_errors; uint64_t errors, syncs; int disagree; } qs_ctx;

static int qs_vote_cond(qs_ctx* q, const int c[3]) {
    q->syncs++;
    if (q->nc == 1) return c[0];
    if (q->nc == 2) { if (c[0] != c[1]) q->disagree = 1; return c[0]; }
    const int c01 = c[0] == c[1], c02 = c[0] == c[2];
    if (!(c01 && c02)) { q->disagree = 1; if (q->count_errors) q->errors++; }
    if (q->majority) return (c[0] & c[1]) | (c[0] & c[2]) | (c[1] & c[2]);
    return c01 ? c[0] : c[2];
}

static void orc_qsort_unit(const int32_t* in, uint32_t L, uint32_t nc, const orc_fault* f, uint32_t flags,
                           int32_t rep[3][1024], qs_ctx* q) {
    q->nc = (int)nc; q->majority = (flags & ORC_F_MAJORITY) != 0; q->count_errors = (flags & ORC_F_COUNT_ERRORS) != 0;
    q->errors = q->syncs = 0; q->disagree = 0;
    for (uint32_t r = 0; r < nc; ++r) memcpy(rep[r], in, 4u * L);
    const int has = f && f->active;
    if (has && f->site >= 32u * L) rep[f->replica][f->site - 32u * L] ^= (int32_t)(1u << f->bit);
    uint32_t ev = 0;                                         /* dynamic index of the next data comparison */
    uint32_t stack_off[1024], stack_len[1024]; int sp = 0;
    stack_off[0] = 0; stack_len[0] = L; sp = 1;
    while (sp > 0) {
        --sp;
        const uint32_t off = stack_off[sp], len = stack_len[sp];
        q->syncs++;                                          /* `if (len < 2) return;` -- indices are never faulted, always agree */
        if (len < 2) continue;
        int32_t pivot[3];
        for (uint32_t r = 0; r < nc; ++r) pivot[r] = rep[r][off + len / 2];              /* :123 */
        int32_t i = 0, j = (int32_t)len - 1;
        for (;; i++, j--) {                                  /* :125 */
            for (;;) {                                       /* while (A[i] < pivot) i++;  :126 */
                int c[3] = {0, 0, 0};
                for (uint32_t r = 0; r < nc; ++r) {
                    int32_t v = rep[r][off + i];
                    if (has && f->replica == r && f->site == ev) v ^= (int32_t)(1u << f->bit);
                    c[r] = v < pivot[r];
                }
                if (i >= (int32_t)len - 1) c[0] = c[1] = c[2] = 0;   /* trap guard: a mis-steered scan stops at the partition edge
                                                                        (on the reference target it would run off the array) */
                ++ev;
                if (!qs_vote_cond(q, c)) break;
                i++;
            }
            for (;;) {                                       /* while (A[j] > pivot) j--;  :127 */
                int c[3] = {0, 0, 0};
                for (uint32_t r = 0; r < nc; ++r) {
                    int32_t v = rep[r][off + j];
                    if (has && f->replica == r && f->site == ev) v ^= (int32_t)(1u << f->bit);
                    c[r] = v > pivot[r];
                }
                if (j <= 0) c[0] = c[1] = c[2] = 0;                   /* trap guard */
                ++ev;
                if (!qs_vote_cond(q, c)) break;
                j--;
            }
            q->syncs++;                                      /* if (i >= j) break;  :128 */
            if (i >= j) break;
            for (uint32_t r = 0; r < nc; ++r) {              /* :129-131, each replica in its own copy */
                int32_t t = rep[r][off + i]; rep[r][off + i] = rep[r][off + j]; rep[r][off + j] = t;
            }
        }
        if (i < 1) i = 1;                                    /* progress guard (only reachable through a mis-steered partition) */
        if (i > (int32_t)len - 1) i = (int32_t)len - 1;
        /* quick_sort(A, i); quick_sort(A + i, len - i);  -- left first: push right, then left */
        stack_off[sp] = off + (uint32_t)i; stack_len[sp] = len - (uint32_t)i; ++sp;
        stack_off[sp] = off; stack_len[sp] = (uint32_t)i; ++sp;
    }
}

/* ------------------------------------------------------------------ */
/* a9-a13: the protected region                                          */
/* ------------------------------------------------------------------ */
/* TMR voter, identical shape at all four sites (synchronization.cpp:439-448,
 * 512-522, 631-642, 934-938):  cmp = (orig == clone1); vote = select cmp, orig, clone2.
 * NOT a bitwise majority.  Error counter (insertTMRCorrectionCount :1354-1465):
 * cmp2 = (orig == clone2) :1391; if !(cmp & cmp2) TMR_ERROR_CNT++ :1400,1428-1431.
 * DWC (splitBlocks :1117-1192): if (orig != clone1) -> FAULT_DETECTED_DWC (:1299-1302). */
static int elem_eq(const uint8_t* a, const uint8_t* b, uint32_t es, int is_float) {
    if (is_float) { float x, y; memcpy(&x, a, 4); memcpy(&y, b, 4); return x == y; } /* fcmp oeq :57-62 */
    return memcmp(a, b, es) == 0;                                                     /* icmp eq */
}

static void run_replica(const orc_desc* d, uint64_t local, const orc_fault* f, uint8_t* out) {
    switch (d->kernel) {
    case ORC_K_CRC16: {
        uint16_t c = orc_crc16((const uint8_t*)d->in + local * d->unit_bytes, d->unit_bytes, f);
        memcpy(out, &c, 2);
    } break;
    case ORC_K_SHA256:
        orc_sha256((const uint8_t*)d->in + local * d->unit_bytes, d->unit_bytes, out, f);
        break;
    case ORC_K_AES128: {
        uint8_t key[16];                       /* each replica mutates ITS copy of key[] (cloneGlobals, cloning.cpp:2417-2462) */
        if (d->mode & ORC_AES_KEY_PER_UNIT) memcpy(key, (const uint8_t*)d->aux + local * 16, 16);
        else memcpy(key, d->key, 16);
        memcpy(out, (const uint8_t*)d->in + local * 16, 16);
        orc_aes128(out, key, (d->mode & ORC_AES_DECRYPT) ? 1 : 0, f);
    } break;
    case ORC_K_MM_U32: {
        uint32_t v = orc_mm_u32_elem((const uint32_t*)d->in, (const uint32_t*)d->aux, d->K, d->N,
                                     (uint32_t)(local / d->N), (uint32_t)(local % d->N), f);
        memcpy(out, &v, 4);
    } break;
    case ORC_K_GEMM_TF32: {
        float v = orc_gemm_tf32_elem((const float*)d->in, (const float*)d->aux, d->K, d->N,
                                     (uint32_t)(local / d->N), (uint32_t)(local % d->N), f);
        memcpy(out, &v, 4);
    } break;
    case ORC_K_CHSTONE_SHA: {
        uint32_t dg[5];
        orc_chstone_sha((const uint8_t*)d->in + local * d->unit_bytes, d->unit_bytes, dg, f);
        memcpy(out, dg, 20);
    } break;
    case ORC_K_CHSTONE_AES: {
        int32_t st[16], key[16];
        memcpy(st, (const uint8_t*)d->in + local * 64, 64);
        if (d->mode & ORC_AES_KEY_PER_UNIT) memcpy(key, (const uint8_t*)d->aux + local * 64, 64);
        else for (int i = 0; i < 16; ++i) key[i] = d->key[i];
        orc_chstone_aes(st, key, (d->mode & ORC_AES_DECRYPT) ? 1 : 0, f);
        memcpy(out, st, 64);
    } break;
    default: break;
    }
}

/* ------------------------------------------------------------------ */
/* 8f-1: -storeDataSync / -noMemReplication -- votes INSIDE the loops     */
/* Rule C4 ("the data used in stores is synchronized", passes.rst repl_details; populateSyncPoints                    */
/* synchronization.cpp:197-221: a store of a non-pointer, computed value is a sync point when -storeDataSync is given  */
/* or memory is not replicated; syncStoreInst :476-560 votes the stored value and, under TMR, hands the VOTED value to */
/* all three copies :519-529).  With -noMemReplication (rule D2: variables live once, in ECC-protected memory; loads   */
/* are still executed per replica from that one address, passes.rst) the replicas re-converge at every assignment.     */
/* Granularity here = the C assignments to the DATA variables of the function (x, crc / sum); pointer stores are never */
/* voted (:199-204) and the loop counters are control state the kernels keep uniform (DESIGN.md section 3).            */
/* Address-offset votes (C3/C5, syncGEP :417-470; -noLoadSync / -noStoreAddrSync prune them) need a data-dependent     */
/* index: crc16 has no subscripts and matrix_multiply indexes with loop counters only, so the set is empty for both.   */
/* A flip at a fault site lands on the replica's copy AFTER the assignment's vote (its reloaded register), so it is    */
/* caught by the next vote on a value computed from it.  Unpinned like every mid-computation site (header).           */
/* ------------------------------------------------------------------ */
int orc_store_votes(uint32_t flags) {
    return (flags & (ORC_F_STORE_DATA_SYNC | ORC_F_NO_MEM_REPLICATION)) && !(flags & ORC_F_NO_STORE_DATA_SYNC);
}
int orc_store_votes_supported(uint32_t kernel) { return kernel == ORC_K_CRC16 || kernel == ORC_K_MM_U32 || kernel == ORC_K_SHA256; }

typedef struct { uint32_t nc, flags; uint64_t errors, syncs; int disagree; } sv_ctx;
/* one store vote on v[0..nc) (width <= 32 bits); TMR: every copy continues with the voted value */
static void sv_vote(sv_ctx* c, uint32_t v[3]) {
    if (c->nc == 1) return;
    if (c->nc == 2) { if (v[0] != v[1]) c->disagree = 1; return; }
    const int c01 = v[0] == v[1], c02 = v[0] == v[2];
    const uint32_t voted = (c->flags & ORC_F_MAJORITY) ? ((v[0] & v[1]) | (v[0] & v[2]) | (v[1] & v[2])) : (c01 ? v[0] : v[2]);
    if (!(c01 && c02)) { c->disagree = 1; if (c->flags & ORC_F_COUNT_ERRORS) c->errors++; }
    if ((c->flags & ORC_F_COUNT_SYNCS) && (c->flags & ORC_F_COUNT_ERRORS)) c->syncs++;
    v[0] = v[1] = v[2] = voted;
}
static uint16_t sv_crc16_unit(const uint8_t* data, uint32_t len, const orc_fault* f, sv_ctx* c) {
    uint32_t crc[3] = { 0xFFFFu, 0xFFFFu, 0xFFFFu }, x[3] = { 0, 0, 0 };
    for (uint32_t n = 0; n < len; ++n) {
        for (uint32_t r = 0; r < c->nc; ++r) {
            uint8_t b = data[n];                                                    /* per-replica load of the one copy */
            if (f->active && f->replica == r && f->site == len + n) b ^= (uint8_t)(1u << f->bit);
            x[r] = (uint8_t)((crc[r] >> 8) ^ b);                                    /* crc16.c:26 */
        }
        sv_vote(c, x);
        for (uint32_t r = 0; r < c->nc; ++r) x[r] = (uint8_t)(x[r] ^ (x[r] >> 4));  /* :27 */
        sv_vote(c, x);
        for (uint32_t r = 0; r < c->nc; ++r)
            crc[r] = (uint16_t)((uint16_t)(crc[r] << 8) ^ (uint16_t)(x[r] << 12) ^ (uint16_t)(x[r] << 5) ^ (uint16_t)x[r]);   /* :28 */
        sv_vote(c, crc);
        for (uint32_t r = 0; r < c->nc; ++r)
            if (f->active && f->replica == r && f->site == n) crc[r] ^= (1u << f->bit);
    }
    sv_vote(c, crc);                                                                /* :30 the SoR exit */
    return (uint16_t)crc[0];
}
static uint32_t sv_mm_elem(const uint32_t* A, const uint32_t* B, uint32_t K, uint32_t N, uint32_t i, uint32_t j, const orc_fault* f, sv_ctx* c) {
    uint32_t sum[3] = { 0, 0, 0 };
    for (uint32_t k = 0; k < K; ++k) {
        for (uint32_t r = 0; r < c->nc; ++r) sum[r] += A[(size_t)i * K + k] * B[(size_t)k * N + j];   /* mm_common_tmr.c:13 */
        sv_vote(c, sum);
        for (uint32_t r = 0; r < c->nc; ++r)
            if (f->active && f->replica == r && f->site == k) sum[r] ^= (1u << f->bit);
    }
    sv_vote(c, sum);                                                                /* :16 r[i][j] = sum */
    return sum[0];
}
/* sha256_transform / sha256_hash with every assignment to a data variable voted, in the reference's statement order:
 *   ctx_data[k] = data[i]              (sha256_common_tmr.c:120)   one u8 vote per message byte
 *   m[i] = pack(...)  i < 16            (:34-40)                    16 votes
 *   m[i] = SIG1(..) + .. i = 16..63     (:42-58)                    48 votes
 *   a..h = ctx_state[0..7]              (:60-67)                     8 votes
 *   t1, t2, h, g, f, e, d, c, b, a      (:78-87) x 64 rounds       640 votes
 *   ctx_state[j] += a..h                (:90-97)                     8 votes
 *   hash[i] = ...                       (:169-178)                  32 votes (the SoR exit)
 * = len + 720 per compression + 32.  Not voted: stores of constants (padding bytes, the IV: syncStoreInst :507-509) and the
 * control state derived from `len` alone (ctx_datalen, ctx_bitlen and the length bytes copied from it, loop counters).
 * A fault site keeps its meaning (m[w] after the pack; a working variable at the entry of round t; ctx_state[j] after the final
 * add): the flip lands on the replica's copy after that assignment's vote.  A flipped working variable can be voted more than
 * once before it is overwritten (e.g. `b`: in t2 through MAJ, then again in `c = b`), so errors_corrected may exceed injected. */
static void sv_sha_compress(uint32_t st[3][8], uint8_t blkb[64], uint32_t nmsg, uint32_t blk, const orc_fault* f, sv_ctx* c) {
    const uint32_t nc = c->nc;
    const int has = f->active && (f->site / SHA_SITES_PER_BLOCK) == blk;
    const uint32_t s = has ? f->site % SHA_SITES_PER_BLOCK : 0xFFFFFFFFu, mask = has ? (1u << f->bit) : 0u, fr = f->replica;
    uint32_t m[3][64], v[3][8], x[3];
    for (uint32_t k = 0; k < nmsg; ++k) { for (uint32_t r = 0; r < 3; ++r) x[r] = blkb[k]; sv_vote(c, x); }      /* :120 */
    for (int i = 0; i < 16; ++i) {
        for (uint32_t r = 0; r < 3; ++r)
            x[r] = ((uint32_t)blkb[4 * i] << 24) | ((uint32_t)blkb[4 * i + 1] << 16) | ((uint32_t)blkb[4 * i + 2] << 8) | (uint32_t)blkb[4 * i + 3];
        sv_vote(c, x);
        for (uint32_t r = 0; r < 3; ++r) m[r][i] = x[r];
        if (s == (uint32_t)i && fr < nc) m[fr][i] ^= mask;
    }
    for (int i = 16; i < 64; ++i) {
        for (uint32_t r = 0; r < 3; ++r) {
            const uint32_t a = m[r][i - 2], b = m[r][i - 15];
            x[r] = (rotr32(a, 17) ^ rotr32(a, 19) ^ (a >> 10)) + m[r][i - 7] + (rotr32(b, 7) ^ rotr32(b, 18) ^ (b >> 3)) + m[r][i - 16];
        }
        sv_vote(c, x);
        for (uint32_t r = 0; r < 3; ++r) m[r][i] = x[r];
    }
    for (int i = 0; i < 8; ++i) {
        for (uint32_t r = 0; r < 3; ++r) x[r] = st[r][i];
        sv_vote(c, x);
        for (uint32_t r = 0; r < 3; ++r) v[r][i] = x[r];
    }
    for (uint32_t t = 0; t < 64; ++t) {
        if (s >= 16u && s < 528u && (s - 16u) / 8u == t && fr < nc) v[fr][(s - 16u) % 8u] ^= mask;
        uint32_t t1[3], t2[3];
        for (uint32_t r = 0; r < 3; ++r) {
            const uint32_t e = v[r][4], ff = v[r][5], g = v[r][6];
            t1[r] = v[r][7] + (rotr32(e, 6) ^ rotr32(e, 11) ^ rotr32(e, 25)) + ((e & ff) ^ (~e & g)) + SHA_K[t] + m[r][t];
        }
        sv_vote(c, t1);
        for (uint32_t r = 0; r < 3; ++r) {
            const uint32_t a = v[r][0], b = v[r][1], cc = v[r][2];
            t2[r] = (rotr32(a, 2) ^ rotr32(a, 13) ^ rotr32(a, 22)) + ((a & b) ^ (a & cc) ^ (b & cc));
        }
        sv_vote(c, t2);
        /* h = g; g = f; f = e; e = d + t1; d = c; c = b; b = a; a = t1 + t2 -- each store voted, in this order */
        for (uint32_t r = 0; r < 3; ++r) x[r] = v[r][6];
        sv_vote(c, x); for (uint32_t r = 0; r < 3; ++r) v[r][7] = x[r];
        for (uint32_t r = 0; r < 3; ++r) x[r] = v[r][5];
        sv_vote(c, x); for (uint32_t r = 0; r < 3; ++r) v[r][6] = x[r];
        for (uint32_t r = 0; r < 3; ++r) x[r] = v[r][4];
        sv_vote(c, x); for (uint32_t r = 0; r < 3; ++r) v[r][5] = x[r];
        for (uint32_t r = 0; r < 3; ++r) x[r] = v[r][3] + t1[r];
        sv_vote(c, x); for (uint32_t r = 0; r < 3; ++r) v[r][4] = x[r];
        for (uint32_t r = 0; r < 3; ++r) x[r] = v[r][2];
        sv_vote(c, x); for (uint32_t r = 0; r < 3; ++r) v[r][3] = x[r];
        for (uint32_t r = 0; r < 3; ++r) x[r] = v[r][1];
        sv_vote(c, x); for (uint32_t r = 0; r < 3; ++r) v[r][2] = x[r];
        for (uint32_t r = 0; r < 3; ++r) x[r] = v[r][0];
        sv_vote(c, x); for (uint32_t r = 0; r < 3; ++r) v[r][1] = x[r];
        for (uint32_t r = 0; r < 3; ++r) x[r] = t1[r] + t2[r];
        sv_vote(c, x); for (uint32_t r = 0; r < 3; ++r) v[r][0] = x[r];
    }
    for (int i = 0; i < 8; ++i) {
        for (uint32_t r = 0; r < 3; ++r) x[r] = st[r][i] + v[r][i];
        sv_vote(c, x);
        for (uint32_t r = 0; r < 3; ++r) st[r][i] = x[r];
        if (s == 528u + (uint32_t)i && fr < nc) st[fr][i] ^= mask;
    }
}
static void sv_sha256_unit(const uint8_t* data, uint32_t len, uint8_t digest[32], const orc_fault* f, sv_ctx* c) {
    uint32_t st[3][8];
    for (uint32_t r = 0; r < 3; ++r) {
        static const uint32_t iv[8] = { 0x6a09e667u, 0xbb67ae85u, 0x3c6ef372u, 0xa54ff53au, 0x510e527fu, 0x9b05688cu, 0x1f83d9abu, 0x5be0cd19u };
        memcpy(st[r], iv, sizeof iv);
    }
    uint8_t buf[64];
    uint32_t blk = 0, off = 0;
    while (len - off >= 64u) { memcpy(buf, data + off, 64); sv_sha_compress(st, buf, 64u, blk++, f, c); off += 64u; }
    const uint32_t rem = len - off;
    memcpy(buf, data + off, rem);
    buf[rem] = 0x80;
    if (rem < 56u) {
        memset(buf + rem + 1, 0, 55u - rem);
    } else {
        memset(buf + rem + 1, 0, 63u - rem);
        sv_sha_compress(st, buf, rem, blk++, f, c);
        memset(buf, 0, 56);
    }
    const uint64_t bits = (uint64_t)len * 8u;
    for (int i = 0; i < 8; ++i) buf[63 - i] = (uint8_t)(bits >> (8 * i));
    sv_sha_compress(st, buf, rem < 56u ? rem : 0u, blk++, f, c);
    for (int w = 0; w < 8; ++w)
        for (int i = 0; i < 4; ++i) {                                   /* :169-178, the SoR exit: one u8 vote per digest byte */
            uint32_t x[3];
            for (uint32_t r = 0; r < 3; ++r) x[r] = (st[r][w] >> (24 - 8 * i)) & 0xFFu;
            sv_vote(c, x);
            digest[4 * w + i] = (uint8_t)x[0];
        }
}
static void sv_run_range(const orc_desc* d, uint64_t u0, uint64_t u1, orc_stats* st) {
    const uint32_t nc = d->num_clones;
    for (uint64_t local = u0; local < u1; ++local) {
        orc_fault f;
        orc_fault_for_unit(d->plan, d->kernel, nc, d->unit_bytes, d->K, d->unit_base + local, local, &f);
        if (f.active) st->injected++;
        sv_ctx c = { nc, d->flags, 0, 0, 0 };
        if (d->kernel == ORC_K_CRC16) {
            uint16_t v = sv_crc16_unit((const uint8_t*)d->in + local * d->unit_bytes, d->unit_bytes, &f, &c);
            memcpy((uint8_t*)d->out + local * 2, &v, 2);
        } else if (d->kernel == ORC_K_SHA256) {
            sv_sha256_unit((const uint8_t*)d->in + local * d->unit_bytes, d->unit_bytes, (uint8_t*)d->out + local * 32, &f, &c);
        } else {
            uint32_t v = sv_mm_elem((const uint32_t*)d->in, (const uint32_t*)d->aux, d->K, d->N, (uint32_t)(local / d->N), (uint32_t)(local % d->N), &f, &c);
            memcpy((uint8_t*)d->out + local * 4, &v, 4);
        }
        st->errors_corrected += c.errors; st->syncs += c.syncs;
        if (nc == 2 && c.disagree) st->dwc_detected++;
        if (c.disagree && d->unit_base + local < st->first_fault_unit) st->first_fault_unit = d->unit_base + local;
    }
}

int orc_run_range(const orc_desc* d, uint64_t u0, uint64_t u1, orc_stats* st) {
    if (!d || d->num_clones < 1 || d->num_clones > 3 || d->kernel >= ORC_K_COUNT_) return -1;
    if (d->kernel == ORC_K_CHSTONE_SHA && (d->unit_bytes < 64u || (d->unit_bytes & 63u) || d->unit_bytes >= (1u << 29))) return -1;
    if (d->kernel == ORC_K_QSORT) {
        const uint32_t L = d->unit_bytes / 4u, nc = d->num_clones;
        if (L < 1 || L > 1024 || (d->unit_bytes & 3u)) return -1;
        static __thread int32_t rep[3][1024];
        for (uint64_t local = u0; local < u1; ++local) {
            orc_fault f;
            orc_fault_for_unit(d->plan, d->kernel, nc, d->unit_bytes, d->K, d->unit_base + local, local, &f);
            if (f.active) st->injected++;
            qs_ctx q;
            orc_qsort_unit((const int32_t*)d->in + local * L, L, nc, &f, d->flags, rep, &q);
            int32_t* out = (int32_t*)d->out + local * L;
            int disagree = q.disagree;
            uint64_t errors = q.errors;
            for (uint32_t e = 0; e < L; ++e) {                  /* SoR exit: one vote per stored element */
                const int32_t r0 = rep[0][e], r1 = nc > 1 ? rep[1][e] : r0, r2 = nc > 2 ? rep[2][e] : r0;
                int32_t v = r0;
                if (nc == 2 && r0 != r1) disagree = 1;
                if (nc == 3) {
                    const int c01 = r0 == r1, c02 = r0 == r2;
                    v = (d->flags & ORC_F_MAJORITY) ? ((r0 & r1) | (r0 & r2) | (r1 & r2)) : (c01 ? r0 : r2);
                    if (!(c01 && c02)) { disagree = 1; if (d->flags & ORC_F_COUNT_ERRORS) errors++; }
                }
                out[e] = v;
            }
            if (nc == 3) {
                st->errors_corrected += errors;
                if ((d->flags & ORC_F_COUNT_SYNCS) && (d->flags & ORC_F_COUNT_ERRORS)) st->syncs += q.syncs + L;
            } else if (nc == 2 && disagree) st->dwc_detected++;
            if (nc > 1 && disagree && d->unit_base + local < st->first_fault_unit) st->first_fault_unit = d->unit_base + local;
        }
        return 0;
    }
    if (orc_store_votes(d->flags) && orc_store_votes_supported(d->kernel)) { sv_run_range(d, u0, u1, st); return 0; }
    const uint32_t ob = orc_out_bytes_per_unit(d->kernel);
    const uint32_t nv = orc_votes_per_unit(d->kernel);
    const uint32_t es = ob / nv;
    const int is_float = d->kernel == ORC_K_GEMM_TF32;
    const uint32_t nc = d->num_clones;
    const orc_fault none = { 0, 0, 0, 0 };
    for (uint64_t local = u0; local < u1; ++local) {
        orc_fault f;
        orc_fault_for_unit(d->plan, d->kernel, nc, d->unit_bytes, d->K, d->unit_base + local, local, &f);
        if (f.active) st->injected++;
        uint8_t rep[3][64];
        for (uint32_t r = 0; r < nc; ++r) run_replica(d, local, (f.active && f.replica == r) ? &f : &none, rep[r]);
        uint8_t* out = (uint8_t*)d->out + local * ob;
        int disagree = 0;
        if (nc == 1) {
            memcpy(out, rep[0], ob);
        } else if (nc == 2) {
            for (uint32_t e = 0; e < nv; ++e)
                if (!elem_eq(rep[0] + e * es, rep[1] + e * es, es, is_float)) disagree = 1;
            memcpy(out, rep[0], ob);            /* compare passes -> the original's store proceeds */
            if (disagree) st->dwc_detected++;
        } else {
            for (uint32_t e = 0; e < nv; ++e) {
                const uint8_t *r0 = rep[0] + e * es, *r1 = rep[1] + e * es, *r2 = rep[2] + e * es;
                int c01 = elem_eq(r0, r1, es, is_float), c02 = elem_eq(r0, r2, es, is_float);
                if (d->flags & ORC_F_MAJORITY) {
                    for (uint32_t b = 0; b < es; ++b)
                        out[e * es + b] = (uint8_t)((r0[b] & r1[b]) | (r0[b] & r2[b]) | (r1[b] & r2[b]));
                } else {
                    memcpy(out + e * es, c01 ? r0 : r2, es);
                }
                if (!(c01 && c02)) {
                    disagree = 1;
                    if (d->flags & ORC_F_COUNT_ERRORS) st->errors_corrected++;
                }
            }
            /* __SYNC_COUNT++ is emitted inside insertTMRCorrectionCount (:1415-1425), i.e. only
             * for TMR with -countErrors. */
            if ((d->flags & ORC_F_COUNT_SYNCS) && (d->flags & ORC_F_COUNT_ERRORS)) st->syncs += nv;
        }
        if (disagree && d->unit_base + local < st->first_fault_unit) st->first_fault_unit = d->unit_base + local;
    }
    return 0;
}

int orc_run(const orc_desc* d, orc_stats* st) { return orc_run_range(d, 0, d ? d->n_units : 0, st); }

typedef struct { const orc_desc* d; uint64_t u0, u1; orc_stats st; int rc; } mt_arg;
static void* mt_main(void* p) {
    mt_arg* a = (mt_arg*)p;
    a->rc = orc_run_range(a->d, a->u0, a->u1, &a->st);
    return NULL;
}
int orc_run_mt(const orc_desc* d, int n_threads, orc_stats* st) {
    if (n_threads < 1) n_threads = 1;
    if (n_threads > 256) n_threads = 256;
    pthread_once(&aes_once, aes_tables);
    pthread_t th[256]; mt_arg args[256];
    uint64_t per = (d->n_units + (uint64_t)n_threads - 1) / (uint64_t)n_threads;
    for (int t = 0; t < n_threads; ++t) {
        uint64_t u0 = per * (uint64_t)t, u1 = u0 + per;
        if (u0 > d->n_units) u0 = d->n_units;
        if (u1 > d->n_units) u1 = d->n_units;
        args[t].d = d; args[t].u0 = u0; args[t].u1 = u1; args[t].rc = 0;
        memset(&args[t].st, 0, sizeof(orc_stats)); args[t].st.first_fault_unit = ~(uint64_t)0;
        pthread_create(&th[t], NULL, mt_main, &args[t]);
    }
    int rc = 0;
    for (int t = 0; t < n_threads; ++t) {
        pthread_join(th[t], NULL);
        if (args[t].rc) rc = args[t].rc;
        st->errors_corrected += args[t].st.errors_corrected;
        st->dwc_detected += args[t].st.dwc_detected;
        st->syncs += args[t].st.syncs;
        st->injected += args[t].st.injected;
        if (args[t].st.first_fault_unit < st->first_fault_unit) st->first_fault_unit = args[t].st.first_fault_unit;
    }
    return rc;
}
