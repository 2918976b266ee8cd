// ORACLE — TEST INFRASTRUCTURE ONLY. Nothing under oracle/ is part of the product
// path; only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline /
// --impl reference legs may build, link or call it.
//
// CPU restatement of the third-party RNG behaviour the reference's results depend
// on. The crate is NOT vendored in the arroy crate; what is restated here is the
// published algorithm of:
//   rand 0.8.5        (Cargo.toml:23)   StdRng, Rng::gen, gen_range, seq::index::sample
//   rand_chacha 0.3.x (transitive)      ChaCha12Rng block layout, 4-block buffer
//   rand_core 0.6.x   (transitive)      BlockRng::next_u32/next_u64, seed_from_u64
// Reference call sites that pin it: src/writer.rs:575, :795, :1128-1133, :1576;
// src/parallel.rs:343, :361; src/lib.rs:134-140; src/tests/mod.rs:105-107.
// Pinned by golden vectors (tests/golden): the f32 stream from seed [42;32]
// (snapshot item values, src/tests/upgrade.rs:117), from_seed(rng.gen()),
// index::sample, u32 gen_range (all build snapshots). seed_from_u64 and gen::<bool>
// have no golden in the reference => "parity unpinned" for those two.
#pragma once
#include <cstdint>
#include <cstring>
#include <vector>

namespace oracle {

static inline uint32_t rotl32(uint32_t x, int k) { return (x << k) | (x >> (32 - k)); }

// One ChaCha block with 12 rounds (6 double rounds), 64-bit block counter in words
// 12/13, stream id 0 in words 14/15 (rand_chacha's layout).
static inline void chacha12_block(const uint32_t key[8], uint64_t counter, uint32_t out[16]) {
    uint32_t s[16] = {0x61707865u, 0x3320646eu, 0x79622d32u, 0x6b206574u,
                      key[0], key[1], key[2], key[3], key[4], key[5], key[6], key[7],
                      (uint32_t)counter, (uint32_t)(counter >> 32), 0u, 0u};
    uint32_t x[16];
    memcpy(x, s, sizeof x);
#define ORACLE_QR(a, b, c, d)                                  \
    x[a] += x[b]; x[d] ^= x[a]; x[d] = rotl32(x[d], 16);       \
    x[c] += x[d]; x[b] ^= x[c]; x[b] = rotl32(x[b], 12);       \
    x[a] += x[b]; x[d] ^= x[a]; x[d] = rotl32(x[d], 8);        \
    x[c] += x[d]; x[b] ^= x[c]; x[b] = rotl32(x[b], 7);
    for (int r = 0; r < 6; ++r) {
        ORACLE_QR(0, 4, 8, 12) ORACLE_QR(1, 5, 9, 13) ORACLE_QR(2, 6, 10, 14) ORACLE_QR(3, 7, 11, 15)
        ORACLE_QR(0, 5, 10, 15) ORACLE_QR(1, 6, 11, 12) ORACLE_QR(2, 7, 8, 13) ORACLE_QR(3, 4, 9, 14)
    }
#undef ORACLE_QR
    for (int i = 0; i < 16; ++i) out[i] = x[i] + s[i];
}

// rand::rngs::StdRng (0.8.5) = ChaCha12Rng behind rand_core::block::BlockRng with a
// 64-word (4-block) result buffer.
struct StdRng {
    uint32_t key[8];
    uint64_t counter;  // next block to generate
    uint32_t buf[64];
    int index;  // 64 == exhausted

    static StdRng from_seed(const uint8_t seed[32]) {
        StdRng r;
        for (int i = 0; i < 8; ++i)
            r.key[i] = (uint32_t)seed[4 * i] | ((uint32_t)seed[4 * i + 1] << 8) |
                       ((uint32_t)seed[4 * i + 2] << 16) | ((uint32_t)seed[4 * i + 3] << 24);
        r.counter = 0;
        r.index = 64;
        return r;
    }

    // rand_core 0.6 SeedableRng::seed_from_u64 (PCG32 expansion). UNPINNED: the
    // reference holds no golden for it (used by examples and src/writer.rs:1133 only).
    static StdRng seed_from_u64(uint64_t state) {
        const uint64_t MUL = 6364136223846793005ull, INC = 11634580027462260723ull;
        uint8_t seed[32];
        for (int c = 0; c < 8; ++c) {
            state = state * MUL + INC;
            uint32_t xorshifted = (uint32_t)(((state >> 18) ^ state) >> 27);
            uint32_t rot = (uint32_t)(state >> 59);
            uint32_t x = (xorshifted >> rot) | (xorshifted << ((32 - rot) & 31));
            seed[4 * c] = (uint8_t)x; seed[4 * c + 1] = (uint8_t)(x >> 8);
            seed[4 * c + 2] = (uint8_t)(x >> 16); seed[4 * c + 3] = (uint8_t)(x >> 24);
        }
        return from_seed(seed);
    }

    void refill() {
        for (int b = 0; b < 4; ++b) chacha12_block(key, counter + b, buf + 16 * b);
        counter += 4;
        index = 0;
    }
    uint32_t next_u32() {
        if (index >= 64) refill();
        return buf[index++];
    }
    // BlockRng::next_u64: two consecutive words of the stream, low word first, also
    // across a buffer refill.
    uint64_t next_u64() {
        uint32_t lo = next_u32();
        uint32_t hi = next_u32();
        return (uint64_t)lo | ((uint64_t)hi << 32);
    }
    // Standard distributions of rand 0.8.5
    float gen_f32() { return (float)(next_u32() >> 8) * (1.0f / 16777216.0f); }
    uint8_t gen_u8() { return (uint8_t)next_u32(); }
    bool gen_bool() { return (int32_t)next_u32() < 0; }  // UNPINNED (no golden)
    void gen_seed(uint8_t out[32]) { for (int i = 0; i < 32; ++i) out[i] = gen_u8(); }
    // StdRng::from_seed(rng.gen())  — src/writer.rs:575, :795
    StdRng fork() { uint8_t s[32]; gen_seed(s); return from_seed(s); }

    // UniformInt<u32>::sample_single_inclusive(low, high)
    uint32_t gen_range_u32_incl(uint32_t low, uint32_t high) {
        uint32_t range = high - low + 1u;
        if (range == 0) return next_u32();
        uint32_t zone = (range << __builtin_clz(range)) - 1u;
        for (;;) {
            uint32_t v = next_u32();
            uint64_t m = (uint64_t)v * (uint64_t)range;
            if ((uint32_t)m <= zone) return low + (uint32_t)(m >> 32);
        }
    }
    // UniformInt<u64>::sample_single(low, high)  (half-open)  — src/writer.rs:1576
    uint64_t gen_range_u64(uint64_t low, uint64_t high) {
        uint64_t range = (high - 1) - low + 1ull;
        if (range == 0) return next_u64();
        uint64_t zone = (range << __builtin_clzll(range)) - 1ull;
        for (;;) {
            uint64_t v = next_u64();
            unsigned __int128 m = (unsigned __int128)v * (unsigned __int128)range;
            if ((uint64_t)m <= zone) return low + (uint64_t)(m >> 64);
        }
    }
    // rand::seq::index::sample(rng, length, 2): amount 2 always takes Floyd's
    // fully-shuffled branch — src/parallel.rs:343
    void sample2(uint32_t length, uint32_t out[2]) {
        std::vector<uint32_t> indices;
        for (uint32_t j = length - 2; j < length; ++j) {
            uint32_t t = gen_range_u32_incl(0, j);
            bool found = false;
            for (size_t p = 0; p < indices.size(); ++p)
                if (indices[p] == t) { indices.insert(indices.begin() + p, j); found = true; break; }
            if (!found) indices.push_back(t);
        }
        out[0] = indices[0];
        out[1] = indices[1];
    }
};

}  // namespace oracle
