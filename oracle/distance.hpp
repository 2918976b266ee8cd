// ORACLE — TEST INFRASTRUCTURE ONLY (see rng.hpp header).
//
// CPU restatement of the reference's arithmetic for the distance / split path:
//   src/spaces/simple.rs:19-83        dispatch AVX(len>=32) -> SSE(len>=16) -> scalar
//   src/spaces/simple_avx.rs:6-110    hsum256, euclid/dot with 4 ymm accumulators + FMA
//   src/spaces/simple_sse.rs:9-110    hsum128, euclid/dot with 4 xmm accumulators, no FMA
//   src/distance/mod.rs:54-110        non_built_distance, normalized_distance, pq_distance,
//                                     norm, normalize, update_mean, side
//   src/distance/mod.rs:126-171       two_means
//   src/distance/{euclidean,cosine,dot_product,manhattan}.rs   the four Distance impls
// Parity target: x86_64 with AVX+FMA detected (the class of host the reference runs on
// next to a GPU). Compile with -mavx2 -mfma -ffp-contract=off: Rust never contracts
// a*b+c, so every non-intrinsic mul/add below must stay separately rounded.
#pragma once
#include <immintrin.h>

#include <cfloat>
#include <cmath>
#include <cstdint>
#include <vector>

#include "rng.hpp"

namespace oracle {

enum Metric : int { EUCLIDEAN = 0, COSINE = 1, DOT_PRODUCT = 2, MANHATTAN = 3,
                    // binary-quantized distances (src/distance/binary_quantized_{euclidean,cosine,manhattan}.rs). Their vectors are
                    // bit strings (src/unaligned_vector/binary_quantized.rs); this restatement keeps them DEQUANTIZED, as the +-1.0
                    // values BinaryQuantized::iter yields (bit 1 -> 1.0, bit 0 -> -1.0), 64 * ceil(dims / 64) of them: a partial last
                    // word is padded with 0 bits = -1.0 and the reference's byte-wise kernels do count those bits.
                    BQ_EUCLIDEAN = 4, BQ_COSINE = 5, BQ_MANHATTAN = 6 };
static inline bool is_bq(int m) { return m >= BQ_EUCLIDEAN; }
static inline int base_metric(int m) { return m == BQ_EUCLIDEAN ? EUCLIDEAN : m == BQ_COSINE ? COSINE : m == BQ_MANHATTAN ? MANHATTAN : m; }

static inline const char* metric_name(int m) {
    switch (m) {  // euclidean.rs:37, cosine.rs:35, dot_product.rs:43, manhattan.rs:36
        case EUCLIDEAN: return "euclidean";
        case COSINE: return "cosine";
        case DOT_PRODUCT: return "dot-product";
        default: return "manhattan";
    }
}
static inline int header_floats(int m) { return m == DOT_PRODUCT ? 2 : 1; }

// BinaryQuantized::from_slice (binary_quantized.rs:80-92) followed by ::iter (:276-289): bit = is_sign_positive(x) (so +0.0 and
// +NaN are 1, -0.0 is 0), value = bit * 2 - 1; `out` has 64 * ceil(d / 64) entries.
static inline size_t bq_padded_dims(size_t d) { return (d + 63) / 64 * 64; }
static inline void bq_quantize_pm1(const float* in, size_t d, float* out) {
    const size_t dp = bq_padded_dims(d);
    for (size_t i = 0; i < dp; ++i) out[i] = (i < d && !std::signbit(in[i])) ? 1.0f : -1.0f;
}
// dot_product_binary_quantized (src/spaces/simple.rs:121-131): per byte count_ones(!(u ^ v)) - count_zeros(..), summed as i32
static inline float dot_bq(const float* a, const float* b, size_t dp) {
    int32_t s = 0;
    for (size_t i = 0; i < dp; ++i) s += ((a[i] > 0.f) == (b[i] > 0.f)) ? 1 : -1;
    return (float)s;
}
static inline uint32_t xor_ones_bq(const float* a, const float* b, size_t dp) {
    uint32_t c = 0;
    for (size_t i = 0; i < dp; ++i) c += ((a[i] > 0.f) != (b[i] > 0.f)) ? 1u : 0u;
    return c;
}

// ---- src/spaces ------------------------------------------------------------------

static inline float hsum256_ps_avx(__m256 x) {  // simple_avx.rs:6-13
    __m128 x128 = _mm_add_ps(_mm256_extractf128_ps(x, 1), _mm256_castps256_ps128(x));
    __m128 x64 = _mm_add_ps(x128, _mm_movehl_ps(x128, x128));
    __m128 x32 = _mm_add_ss(x64, _mm_shuffle_ps(x64, x64, 0x55));
    return _mm_cvtss_f32(x32);
}
static inline float hsum128_ps_sse(__m128 x) {  // simple_sse.rs:9-14
    __m128 x64 = _mm_add_ps(x, _mm_movehl_ps(x, x));
    __m128 x32 = _mm_add_ss(x64, _mm_shuffle_ps(x64, x64, 0x55));
    return _mm_cvtss_f32(x32);
}

static inline float dot_avx(const float* a, const float* b, size_t n) {  // simple_avx.rs:67-110
    size_t m = n - (n % 32);
    __m256 s1 = _mm256_setzero_ps(), s2 = s1, s3 = s1, s4 = s1;
    for (size_t i = 0; i < m; i += 32) {
        s1 = _mm256_fmadd_ps(_mm256_loadu_ps(a + i), _mm256_loadu_ps(b + i), s1);
        s2 = _mm256_fmadd_ps(_mm256_loadu_ps(a + i + 8), _mm256_loadu_ps(b + i + 8), s2);
        s3 = _mm256_fmadd_ps(_mm256_loadu_ps(a + i + 16), _mm256_loadu_ps(b + i + 16), s3);
        s4 = _mm256_fmadd_ps(_mm256_loadu_ps(a + i + 24), _mm256_loadu_ps(b + i + 24), s4);
    }
    float result = hsum256_ps_avx(s1) + hsum256_ps_avx(s2) + hsum256_ps_avx(s3) + hsum256_ps_avx(s4);
    for (size_t i = m; i < n; ++i) result += a[i] * b[i];
    return result;
}
static inline float euclid_avx(const float* a, const float* b, size_t n) {  // simple_avx.rs:15-65
    size_t m = n - (n % 32);
    __m256 s1 = _mm256_setzero_ps(), s2 = s1, s3 = s1, s4 = s1;
    for (size_t i = 0; i < m; i += 32) {
        __m256 d1 = _mm256_sub_ps(_mm256_loadu_ps(a + i), _mm256_loadu_ps(b + i));
        s1 = _mm256_fmadd_ps(d1, d1, s1);
        __m256 d2 = _mm256_sub_ps(_mm256_loadu_ps(a + i + 8), _mm256_loadu_ps(b + i + 8));
        s2 = _mm256_fmadd_ps(d2, d2, s2);
        __m256 d3 = _mm256_sub_ps(_mm256_loadu_ps(a + i + 16), _mm256_loadu_ps(b + i + 16));
        s3 = _mm256_fmadd_ps(d3, d3, s3);
        __m256 d4 = _mm256_sub_ps(_mm256_loadu_ps(a + i + 24), _mm256_loadu_ps(b + i + 24));
        s4 = _mm256_fmadd_ps(d4, d4, s4);
    }
    float result = hsum256_ps_avx(s1) + hsum256_ps_avx(s2) + hsum256_ps_avx(s3) + hsum256_ps_avx(s4);
    for (size_t i = m; i < n; ++i) { float t = a[i] - b[i]; result += t * t; }  // powi(2)
    return result;
}
static inline float dot_sse(const float* a, const float* b, size_t n) {  // simple_sse.rs:63-110
    size_t m = n - (n % 16);
    __m128 s1 = _mm_setzero_ps(), s2 = s1, s3 = s1, s4 = s1;
    for (size_t i = 0; i < m; i += 16) {
        s1 = _mm_add_ps(_mm_mul_ps(_mm_loadu_ps(a + i), _mm_loadu_ps(b + i)), s1);
        s2 = _mm_add_ps(_mm_mul_ps(_mm_loadu_ps(a + i + 4), _mm_loadu_ps(b + i + 4)), s2);
        s3 = _mm_add_ps(_mm_mul_ps(_mm_loadu_ps(a + i + 8), _mm_loadu_ps(b + i + 8)), s3);
        s4 = _mm_add_ps(_mm_mul_ps(_mm_loadu_ps(a + i + 12), _mm_loadu_ps(b + i + 12)), s4);
    }
    float result = hsum128_ps_sse(s1) + hsum128_ps_sse(s2) + hsum128_ps_sse(s3) + hsum128_ps_sse(s4);
    for (size_t i = m; i < n; ++i) result += a[i] * b[i];
    return result;
}
static inline float euclid_sse(const float* a, const float* b, size_t n) {  // simple_sse.rs:16-61
    size_t m = n - (n % 16);
    __m128 s1 = _mm_setzero_ps(), s2 = s1, s3 = s1, s4 = s1;
    for (size_t i = 0; i < m; i += 16) {
        __m128 d1 = _mm_sub_ps(_mm_loadu_ps(a + i), _mm_loadu_ps(b + i));
        s1 = _mm_add_ps(_mm_mul_ps(d1, d1), s1);
        __m128 d2 = _mm_sub_ps(_mm_loadu_ps(a + i + 4), _mm_loadu_ps(b + i + 4));
        s2 = _mm_add_ps(_mm_mul_ps(d2, d2), s2);
        __m128 d3 = _mm_sub_ps(_mm_loadu_ps(a + i + 8), _mm_loadu_ps(b + i + 8));
        s3 = _mm_add_ps(_mm_mul_ps(d3, d3), s3);
        __m128 d4 = _mm_sub_ps(_mm_loadu_ps(a + i + 12), _mm_loadu_ps(b + i + 12));
        s4 = _mm_add_ps(_mm_mul_ps(d4, d4), s4);
    }
    float result = hsum128_ps_sse(s1) + hsum128_ps_sse(s2) + hsum128_ps_sse(s3) + hsum128_ps_sse(s4);
    for (size_t i = m; i < n; ++i) { float t = a[i] - b[i]; result += t * t; }
    return result;
}
// simple.rs:49-51 / :81-83 — iter().map().sum(); the f32 Sum fold starts at +0.0 on
// the toolchain the reference's CI pins (Rust 1.82, .github/workflows/rust.yml:26).
static inline float dot_scalar(const float* a, const float* b, size_t n) {
    float s = 0.0f;
    for (size_t i = 0; i < n; ++i) s += a[i] * b[i];
    return s;
}
static inline float euclid_scalar(const float* a, const float* b, size_t n) {
    float s = 0.0f;
    for (size_t i = 0; i < n; ++i) s += (a[i] - b[i]) * (a[i] - b[i]);
    return s;
}
static inline float dot_product(const float* a, const float* b, size_t n) {  // simple.rs:53-79
    if (n >= 32) return dot_avx(a, b, n);
    if (n >= 16) return dot_sse(a, b, n);
    return dot_scalar(a, b, n);
}
static inline float euclidean_distance(const float* a, const float* b, size_t n) {  // simple.rs:19-45
    if (n >= 32) return euclid_avx(a, b, n);
    if (n >= 16) return euclid_sse(a, b, n);
    return euclid_scalar(a, b, n);
}

// ---- src/distance ----------------------------------------------------------------

// A borrowed leaf: header + vector. Header layout per metric (node.rs:68-73):
//   Euclidean / Manhattan {bias}            -> h0
//   Cosine               {norm}             -> h0
//   DotProduct           {extra_dim, norm}  -> h0, h1      (dot_product.rs:24-29)
struct Leaf {
    float h0, h1;
    const float* v;
};
struct OwnedLeaf {
    float h0 = 0.f, h1 = 0.f;
    std::vector<float> v;
    Leaf view() const { return Leaf{h0, h1, v.data()}; }
};

static inline float norm_no_header(const float* v, size_t d) { return std::sqrt(dot_product(v, v, d)); }

// D::new_header — euclidean.rs:41, cosine.rs:39, dot_product.rs:47, manhattan.rs:40
static inline void new_header(int m, const float* v, size_t d, float& h0, float& h1) {
    h0 = 0.f; h1 = 0.f;
    if (m == COSINE) h0 = norm_no_header(v, d);
    if (m == BQ_COSINE) h0 = std::sqrt(dot_bq(v, v, d));   // binary_quantized_cosine.rs:47-49, :70-72
}

static inline float built_distance(int m, const Leaf& p, const Leaf& q, size_t d) {
    switch (m) {
        case BQ_EUCLIDEAN: return (float)(xor_ones_bq(p.v, q.v, d) * 4u);   // binary_quantized_euclidean.rs:117-124
        case BQ_MANHATTAN: return (float)(xor_ones_bq(p.v, q.v, d) * 2u);   // binary_quantized_manhattan.rs:113-120
        case BQ_COSINE: {                                                   // binary_quantized_cosine.rs:51-65 (no clamp, `!= 0.0`)
            float pn = p.h0, qn = q.h0;
            float pq = dot_bq(p.v, q.v, d);
            float pnqn = pn * qn;
            if (pnqn != 0.0f) { float c = pq / pnqn; return (1.0f - c) / 2.0f; }
            return 0.0f;
        }
        case EUCLIDEAN: return euclidean_distance(p.v, q.v, d);  // euclidean.rs:45-47
        case COSINE: {                                           // cosine.rs:43-59
            float pn = p.h0, qn = q.h0;
            float pq = dot_product(p.v, q.v, d);
            float pnqn = pn * qn;
            if (pnqn > FLT_EPSILON) {
                float c = pq / pnqn;
                // f32::clamp: NaN stays NaN
                if (c < -1.0f) c = -1.0f;
                if (c > 1.0f) c = 1.0f;
                return (1.0f - c) / 2.0f;
            }
            return 0.0f;
        }
        case DOT_PRODUCT: return -dot_product(p.v, q.v, d);  // dot_product.rs:52-56
        default: {                                           // manhattan.rs:44-46
            float s = 0.0f;
            for (size_t i = 0; i < d; ++i) s += std::fabs(p.v[i] - q.v[i]);
            return s;
        }
    }
}
static inline float non_built_distance(int m, const Leaf& p, const Leaf& q, size_t d) {
    if (m != DOT_PRODUCT) return built_distance(m, p, q, d);  // mod.rs:54-56
    // dot_product.rs:58-70
    float pp = p.h1, qq = q.h1;
    float pq = dot_product(p.v, q.v, d) + p.h0 * q.h0;
    float ppqq = pp * qq;
    if (ppqq >= FLT_MIN) return 2.0f - 2.0f * pq / std::sqrt(ppqq);
    return 2.0f;
}
// `dims` = the index' dimensions (Reader::dimensions, reader.rs:398) — only the binary-quantized distances use it
static inline float normalized_distance(int m, float dist, size_t dims = 0) {
    switch (m) {
        case BQ_EUCLIDEAN: return dist / (float)dims;                                               // binary_quantized_euclidean.rs:56-58
        case BQ_MANHATTAN: return ((dist != dist) ? 0.0f : (dist > 0.0f ? dist : 0.0f)) / (float)dims;   // binary_quantized_manhattan.rs:56-58
        case BQ_COSINE: return dist;
        case EUCLIDEAN: return std::sqrt(dist);                    // mod.rs:59-61
        case COSINE: return dist;                                  // cosine.rs:61-63
        case DOT_PRODUCT: return -dist;                            // dot_product.rs:81-83
        default: return (dist != dist) ? 0.0f : (dist > 0.0f ? dist : 0.0f);  // manhattan.rs:48-50 f32::max
    }
}
static inline float norm_leaf(int m, const Leaf& l, size_t d) {
    if (m == BQ_EUCLIDEAN || m == BQ_COSINE) return std::sqrt(dot_bq(l.v, l.v, d));   // norm_no_header of the two
    if (m == BQ_MANHATTAN) { float s = 0.f; for (size_t i = 0; i < d; ++i) s += l.v[i] > 0.f ? 1.f : -1.f; return std::sqrt(s); }   // binary_quantized_manhattan.rs:60-67
    if (m == DOT_PRODUCT) {  // dot_product.rs:72-75
        float dot = dot_product(l.v, l.v, d);
        return std::sqrt(dot + l.h0 * l.h0);
    }
    return norm_no_header(l.v, d);  // mod.rs:70-72
}
static inline void normalize(int m, OwnedLeaf& node, size_t d) {  // mod.rs:76-82, dot_product.rs:85-92
    float norm = norm_leaf(m, node.view(), d);
    if (norm > 0.0f) {
        for (size_t i = 0; i < d; ++i) node.v[i] = node.v[i] / norm;
        if (m == DOT_PRODUCT) node.h0 /= norm;
    }
}
static inline void init_leaf(int m, OwnedLeaf& node, size_t d) {
    if (m == COSINE) node.h0 = std::sqrt(dot_product(node.v.data(), node.v.data(), d));  // cosine.rs:69-71
    else if (m == DOT_PRODUCT) node.h1 = dot_product(node.v.data(), node.v.data(), d);    // dot_product.rs:94-96
}
static inline void update_mean(OwnedLeaf& mean, const Leaf& k, float norm, float c, size_t d) {  // mod.rs:86-94
    for (size_t i = 0; i < d; ++i) mean.v[i] = (mean.v[i] * c + k.v[i] / norm) / (c + 1.0f);
}
static inline float margin(int m, const Leaf& n, const Leaf& q, size_t d) {
    switch (m) {
        case BQ_EUCLIDEAN:
        case BQ_MANHATTAN: return n.h0 + dot_bq(n.v, q.v, d);   // binary_quantized_euclidean.rs:95-97, _manhattan.rs:99-101
        case BQ_COSINE: return dot_bq(n.v, q.v, d);             // binary_quantized_cosine.rs:95-97
        case EUCLIDEAN:
        case MANHATTAN: return n.h0 + dot_product(n.v, q.v, d);   // euclidean.rs:79-81, manhattan.rs:82-84
        case COSINE: return dot_product(n.v, q.v, d);              // cosine.rs:87-89
        default: return dot_product(n.v, q.v, d) + n.h0 * q.h0;    // dot_product.rs:115-117
    }
}
// mod.rs:103-110 — is_sign_positive: +0.0 and +NaN are Right, -0.0 and -NaN are Left.
static inline bool side_is_right(float margin_value) { return !std::signbit(margin_value); }
static inline float pq_distance(float distance, float margin_value, bool right) {  // mod.rs:63-68, f32::min
    float a = right ? margin_value : -margin_value;
    if (a != a) return distance;
    if (distance != distance) return a;
    return a < distance ? a : distance;
}

// The sampler two_means draws from: positions in an ascending id subset
// (ImmutableSubsetLeafs, src/parallel.rs:316-367). `get(pos)` returns the leaf at
// rank pos of the subset.
struct SubsetView {
    const uint32_t* rows;  // ascending row indices (row == rank of the item id)
    uint32_t len;
    const float* vectors;  // n x d, row-major
    const float* h0;
    const float* h1;
    size_t d;
    Leaf get(uint32_t pos) const {
        uint32_t r = rows[pos];
        return Leaf{h0[r], h1 ? h1[r] : 0.f, vectors + (size_t)r * d};
    }
};

// src/distance/mod.rs:126-171
static inline void two_means(int m, StdRng& rng, const SubsetView& leafs, bool cosine, OwnedLeaf& p, OwnedLeaf& q) {
    const size_t d = leafs.d;
    uint32_t idx[2];
    rng.sample2(leafs.len, idx);  // choose_two, parallel.rs:342-353
    Leaf lp = leafs.get(idx[0]), lq = leafs.get(idx[1]);
    p.h0 = lp.h0; p.h1 = lp.h1; p.v.assign(lp.v, lp.v + d);
    q.h0 = lq.h0; q.h1 = lq.h1; q.v.assign(lq.v, lq.v + d);
    if (cosine) { normalize(m, p, d); normalize(m, q, d); }
    init_leaf(m, p, d);
    init_leaf(m, q, d);
    float ic = 1.0f, jc = 1.0f;
    for (int it = 0; it < 10; ++it) {
        uint32_t kpos = rng.gen_range_u32_incl(0, leafs.len - 1);  // choose, parallel.rs:356-367
        Leaf k = leafs.get(kpos);
        float di = ic * non_built_distance(m, p.view(), k, d);
        float dj = jc * non_built_distance(m, q.view(), k, d);
        float norm = cosine ? norm_leaf(m, k, d) : 1.0f;
        if (norm != norm || norm <= 0.0f) continue;
        if (di < dj) {
            update_mean(p, k, norm, ic, d);
            init_leaf(m, p, d);
            ic += 1.0f;
        } else if (dj < di) {
            update_mean(q, k, norm, jc, d);
            init_leaf(m, q, d);
            jc += 1.0f;
        }
    }
}

// D::create_split — euclidean.rs:55-77, manhattan.rs:58-80, cosine.rs:73-85, dot_product.rs:98-113
static inline void create_split(int m, StdRng& rng, const SubsetView& children, OwnedLeaf& normal) {
    const size_t d = children.d;
    OwnedLeaf p, q;
    if (is_bq(m)) {
        // two_means_binary_quantized (mod.rs:173-223): the sampled leaves become f32 leaves of the NON-quantized distance
        // (`new_leaf(vector.to_vec())`: header = NonBq::new_header — the Cosine norm of a +-1 vector is the BQ header's value,
        // the others are 0), then the ordinary loop; the children view already holds exactly those vectors and headers.
        const int nb = base_metric(m);
        two_means(nb, rng, children, m == BQ_COSINE, p, q);
        // create_split (binary_quantized_*.rs): p - q goes through UnalignedVector::<BinaryQuantized>::from_vec = its sign bits.
        // Self::normalize then divides by a positive norm (or does nothing) and re-quantizes: the bits do not change.
        normal.h0 = 0.f; normal.h1 = 0.f;
        normal.v.resize(d);
        for (size_t i = 0; i < d; ++i) normal.v[i] = std::signbit(p.v[i] - q.v[i]) ? -1.0f : 1.0f;
        if (m != BQ_COSINE) {
            // bias = sum of -n * (P + Q) / 2 over the QUANTIZED centroids P, Q (euclidean.rs:83-89)
            float bias = 0.0f;
            for (size_t i = 0; i < d; ++i) {
                const float P = std::signbit(p.v[i]) ? -1.0f : 1.0f, Q = std::signbit(q.v[i]) ? -1.0f : 1.0f;
                bias += -normal.v[i] * (P + Q) / 2.0f;
            }
            normal.h0 = bias;
        }
        return;
    }
    bool cosine = (m == COSINE || m == DOT_PRODUCT);
    two_means(m, rng, children, cosine, p, q);
    normal.h0 = 0.f; normal.h1 = 0.f;
    normal.v.resize(d);
    for (size_t i = 0; i < d; ++i) normal.v[i] = p.v[i] - q.v[i];
    if (m == DOT_PRODUCT) normal.h0 = p.h0 - q.h0;  // extra_dim
    normalize(m, normal, d);
    if (m == EUCLIDEAN || m == MANHATTAN) {
        float bias = 0.0f;  // .sum() over ((-n) * (p + q)) / 2.0
        for (size_t i = 0; i < d; ++i) bias += -normal.v[i] * (p.v[i] + q.v[i]) / 2.0f;
        normal.h0 = bias;
    }
}

}  // namespace oracle
