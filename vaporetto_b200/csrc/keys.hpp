// Record formats, key encoding and hash geometry shared by the host table builder and the kernels.
#pragma once
#include <cstdint>

#include "common.hpp"

namespace vpt {

constexpr uint32_t kNoPattern = 0xFFFFFFFFu;
constexpr int kInlineWidth = 6;  // weights stored inside a 32-byte fast record

// Hash-table geometry shared by host builder and device kernels.  A dense table with 8-bit seeds places most keys in
// its nslots primary slots; the buckets no seed could place there carry kSpillSeed, and their keys live in a sparse
// spill table behind the primary ones (one slot space: slot numbers nslots .. nslots + spill_slots_of(nslots) - 1),
// whose spill_buckets_of(nbuckets) seeds follow the nbuckets primary seeds.
struct TableGeom {
    uint32_t nslots = 0;
    uint32_t nbuckets = 0;
    uint64_t salt = 0;
    uint32_t seed_bits = 8;  // 8: one byte per bucket (fits shared memory); 16: dense tables that live in L2
    bool spill = false;      // the table has a spill table (8-bit seeds only)
};

// 32-byte records.  `key` bit 63 = node has longer extensions (a deeper node exists).
struct alignas(32) FastRecord {
    uint64_t key;
    int32_t w[kInlineWidth];  // boundary weights for relative positions R0 .. R0+5
};
struct alignas(32) GeneralRecord {
    uint64_t key;
    uint32_t pid;      // longest pattern that is a suffix of the node string, or kNoPattern
    uint32_t row_ptr;  // index of the row's first weight in the pool, or kNoPattern
    int32_t off;       // row offset (relative to the matched end char)
    uint32_t len;      // row length
    uint32_t node_id;
    uint32_t pad;
};
static_assert(sizeof(FastRecord) == 32 && sizeof(GeneralRecord) == 32, "record size");

constexpr uint64_t kExtFlag = 1ull << 63;
// Deep keys (depth >= 4) leave bits 59..61 of the key free (their top field is kDeepMarker + a 10-bit value):
// bit 61 marks a record whose merged row does not fit the inline window; the part outside the window lives in
// the overflow pool (slot_ovf side array).  Only deep records can carry it: rows of patterns of <= 3 symbols
// must fit the window for a table to use the inline format at all.
constexpr uint64_t kOvfFlag = 1ull << 61;
constexpr uint64_t kDeepMarker = 0x110000ull;  // first invalid code point: marks (parent node, symbol) keys

// Records of 2-symbol nodes (c1 field of the key unused) carry in that field a 19-bit mask of their 3-symbol
// extensions: bit child_bit(c1) is set for every c1 such that (c1, c2, c3) is a node.  A clear bit proves that the
// 3-symbol node does not exist, so the probe for it is skipped (bits 61 / 62 of the key stay clear).
constexpr int kChildMaskBits = 19;
constexpr uint64_t kChildMaskField = ((1ull << kChildMaskBits) - 1) << 42;

// key of a node at depth <= 3: c3 is the last symbol of the suffix, c1 the first (0 if absent).
VPT_HD uint64_t shallow_key(uint32_t c1, uint32_t c2, uint32_t c3) {
    return (uint64_t(c1) << 42) | (uint64_t(c2) << 21) | uint64_t(c3);
}
// key of a node at depth >= 4: parent node id and the symbol preceding the parent's string.
VPT_HD uint64_t deep_key(uint32_t parent_id, uint32_t sym) {
    return ((kDeepMarker + (uint64_t(parent_id) >> 21)) << 42) | ((uint64_t(parent_id) & 0x1FFFFF) << 21) | uint64_t(sym);
}

// Hash-and-displace perfect hash (32-bit arithmetic: cheap on the GPU).  A key is reduced to two 32-bit hashes
// that are LINEAR in its three 21-bit fields (c1, c2, c3): h = c3*k[0] + c2*k[1] + c1*k[2] (mod 2^32), with odd
// multipliers derived from the table's salt.  Linearity is what the streaming kernel (fused.cu) exploits: the
// hashes of the three suffix levels of one text position share their partial sums (h1 = c3*k0, h2 = h1 + c2*k1,
// h3 = h2 + c1*k2), so a fallback probe costs one multiply-add per hash instead of a full mix.  Every consumer
// reads the HIGH bits of these sums or of a product of them (mulhi32), which depend on all input bits.  The
// builder checks that no two keys of a table share both hashes (it re-salts otherwise).
struct HashK {
    uint32_t a[3];  // bucket hash multipliers for c3, c2, c1
    uint32_t b[3];  // displacement hash multipliers
};
VPT_HD HashK hash_consts(uint64_t salt) {
    HashK k;
    for (int i = 0; i < 3; ++i) {
        const uint64_t m = mix64(salt + 0x9E3779B97F4A7C15ull * uint64_t(i + 1));
        k.a[i] = uint32_t(m) | 1u;
        k.b[i] = uint32_t(m >> 32) | 1u;
    }
    return k;
}
VPT_HD void key_hashes(uint64_t key, const HashK& k, uint32_t& ha, uint32_t& hb) {
    const uint32_t c3 = uint32_t(key) & 0x1FFFFFu, c2 = uint32_t(key >> 21) & 0x1FFFFFu, c1 = uint32_t(key >> 42) & 0x1FFFFFu;
    ha = c3 * k.a[0] + c2 * k.a[1] + c1 * k.a[2];
    hb = c3 * k.b[0] + c2 * k.b[1] + c1 * k.b[2];
}
VPT_HD uint32_t mulhi32(uint32_t a, uint32_t b) {
#ifdef __CUDA_ARCH__
    return __umulhi(a, b);  // one IMAD.HI (the 64-bit form can become a wide product and a shift)
#else
    return uint32_t((uint64_t(a) * b) >> 32);
#endif
}
VPT_HD uint32_t child_bit(uint32_t c1) { return mulhi32(c1 * 0x9E3779B1u, uint32_t(kChildMaskBits)); }
VPT_HD uint32_t bucket_of(uint32_t ha, uint32_t nbuckets) { return mulhi32(ha, nbuckets); }
// The probe rule: key hashes + seeds -> slot.  In a table with a spill table, a primary seed of kSpillSeed (never a
// placing 8-bit seed) sends the key to the spill table: its bucket there is picked by the displacement hash hb
// (spill_bucket_of), it is displaced by kSpillSeed + that bucket's seed with the spill table's own multiplier, into
// slots nslots ...  Both seeds are read before this (the spill seed whether it is needed or not, so that the two
// loads are independent); the spill seed only counts for a spilled bucket.  kSpill = false is the rule of a table
// without a spill table (every seed places; 16-bit seeds); an 8-bit table without one never carries kSpillSeed, so
// kSpill = true serves it too.  The selects are multiply-adds by sp (0 / 1): the kernels' ALU pipe is their busiest
// unit, the FMA pipe is not.
constexpr uint32_t kSpillSeed = 255;
constexpr uint32_t kPrimaryMul = 0x85EBCA6Bu;
// The spill table's geometry follows from the primary one, so that nslots, nbuckets, the salt and the seeds are all a
// prober needs: a third as many slots (about 18 % of a 0.75-load table's keys spill: load ~0.35), an eighth as many
// buckets (8-12 keys each), and a displacement multiplier of its own derived from the salt.
VPT_HD uint32_t spill_slots_of(uint32_t nslots) { return nslots / 3 + 1; }
VPT_HD uint32_t spill_buckets_of(uint32_t nbuckets) { return nbuckets / 8 + 1; }
VPT_HD uint32_t spill_mul(uint64_t salt) { return uint32_t(mix64(salt + 0x9E3779B97F4A7C15ull * 4)) | 1u; }
// index of a key's spill seed in the seed array (the spill seeds follow the nbuckets primary ones)
VPT_HD uint32_t spill_bucket_of(uint32_t hb, uint32_t nbuckets, uint32_t spill_buckets) {
    return mulhi32(hb, spill_buckets) + nbuckets;
}
template <bool kSpill>
VPT_HD uint32_t slot_of_seeds(uint32_t ha, uint32_t hb, uint32_t seed, uint32_t spill_seed, uint32_t nslots,
                              uint32_t spill_slots, uint32_t spill_multiplier) {
    const uint32_t sp = kSpill && seed == kSpillSeed ? 1u : 0u;
    const uint32_t v = (hb + (seed + sp * spill_seed) * (ha | 1u)) * (kPrimaryMul + sp * (spill_multiplier - kPrimaryMul));
    return mulhi32(v, nslots + sp * (spill_slots - nslots)) + sp * nslots;
}

}  // namespace vpt
