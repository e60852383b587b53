/*
 * knn_oracle.c — CPU restatement of NornicDB's brute-force vector-similarity path.
 *
 * THIS IS TEST INFRASTRUCTURE, NOT PRODUCT CODE.  Only tests/, __graft_entry__.smoke()
 * and bench.py's cpu_baseline / --impl reference legs may load it.  The product path
 * (nornicdb_b200/) never links, imports or calls anything in oracle/.
 *
 * Parity pinning: every function below is checked (tests/test_oracle_kat.py) against the
 * literal known-answer vectors of the reference's own tests (SURVEY.md §8c:
 * pkg/simd/simd_test.go, pkg/math/vector/similarity_test.go, pkg/gpu/cuda/cuda_test.go,
 * pkg/gpu/gpu_test.go).  Those tests pin small-d semantics and edge cases only; nothing in
 * the reference pins numeric results at d>=128, so large-shape parity is defined by the
 * fp64 scorer orc_knn_exact64() below.
 *
 * Third-party note: the arithmetic of pkg/simd lives in github.com/viterin/vek v0.4.3
 * (go.mod:17), which is NOT present in the reference repository and cannot be fetched (no Go
 * toolchain, no network).  Its published algorithm is restated here: vek32.Dot = sum a[i]*b[i];
 * vek32.CosineSimilarity = dot / sqrt(sum a^2 * sum b^2) in one pass (NaN for zero vectors,
 * which pkg/simd/simd_amd64.go:31-35 maps to 0); vek32.Distance = sqrt(sum (a-b)^2);
 * vek32.Norm = sqrt(sum v^2).  The same definitions appear in-repo as the pure-Go
 * references of pkg/simd/benchmark_test.go:25-63, which this file follows line for line in
 * sequential fp32.
 *
 * Compile WITHOUT fast-math (oracle/Makefile: -O2 -ffp-contract=off) so fp32 sums are the
 * sequential sums the Go code produces.
 */
#include <float.h>
#include <math.h>
#include <stddef.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#ifdef _OPENMP
#include <omp.h>
#endif

#define ORC_COSINE 0
#define ORC_DOT 1
#define ORC_EUCLIDEAN 2

#define ORC_F32 0
#define ORC_F16 1

/* ---------------------------------------------------------------- pkg/simd ------------- */

/* simd.DotProduct — pkg/simd/simd.go:38-43 (guards), benchmark_test.go:25-31 (definition). */
float orc_dot(const float *a, size_t na, const float *b, size_t nb) {
    if (na != nb || na == 0) return 0.0f;
    float sum = 0.0f;
    for (size_t i = 0; i < na; i++) sum += a[i] * b[i];
    return sum;
}

/* simd.CosineSimilarity — pkg/simd/simd.go:62-67, simd_amd64.go:27-37 (NaN -> 0),
 * benchmark_test.go:33-46 (dot / sqrt(normA*normB), 0 when either norm is 0). */
float orc_cosine(const float *a, size_t na, const float *b, size_t nb) {
    if (na != nb || na == 0) return 0.0f;
    float dot = 0.0f, xa = 0.0f, xb = 0.0f;
    for (size_t i = 0; i < na; i++) {
        dot += a[i] * b[i];
        xa += a[i] * a[i];
        xb += b[i] * b[i];
    }
    float r = dot / (float)sqrt((double)(xa * xb));
    if (isnan(r)) return 0.0f;
    return r;
}

/* simd.EuclideanDistance — pkg/simd/simd.go:83-88, benchmark_test.go:48-55. */
float orc_euclid(const float *a, size_t na, const float *b, size_t nb) {
    if (na != nb || na == 0) return 0.0f;
    float sum = 0.0f;
    for (size_t i = 0; i < na; i++) {
        float diff = a[i] - b[i];
        sum += diff * diff;
    }
    return (float)sqrt((double)sum);
}

/* simd.Norm — pkg/simd/simd.go:98-100, simd_amd64.go:46-51, benchmark_test.go:57-63. */
float orc_norm(const float *v, size_t n) {
    if (n == 0) return 0.0f;
    float sum = 0.0f;
    for (size_t i = 0; i < n; i++) sum += v[i] * v[i];
    return (float)sqrt((double)sum);
}

/* simd.NormalizeInPlace — pkg/simd/simd.go:113-115, simd_amd64.go:53-62 (no-op on zero norm;
 * vek32.DivNumber_Inplace divides each element by the norm). */
void orc_normalize_inplace(float *v, size_t n) {
    if (n == 0) return;
    float nrm = orc_norm(v, n);
    if (nrm == 0.0f) return;
    for (size_t i = 0; i < n; i++) v[i] = v[i] / nrm;
}

/* simd.BatchCosineSimilarity / BatchDotProduct / BatchEuclideanDistance — pkg/simd/simd.go:149-231.
 * embeddings is a contiguous [n_vectors x dims] array; silently returns when scores is too short. */
void orc_batch_cosine(const float *emb, size_t emb_len, const float *q, size_t dims, float *scores,
                      size_t scores_len) {
    if (dims == 0) return;
    size_t n = emb_len / dims;
    if (n == 0 || scores_len < n) return;
    for (size_t i = 0; i < n; i++) scores[i] = orc_cosine(emb + i * dims, dims, q, dims);
}
void orc_batch_dot(const float *emb, size_t emb_len, const float *q, size_t dims, float *scores,
                   size_t scores_len) {
    if (dims == 0) return;
    size_t n = emb_len / dims;
    if (n == 0 || scores_len < n) return;
    for (size_t i = 0; i < n; i++) scores[i] = orc_dot(emb + i * dims, dims, q, dims);
}
void orc_batch_euclid(const float *emb, size_t emb_len, const float *q, size_t dims, float *scores,
                      size_t scores_len) {
    if (dims == 0) return;
    size_t n = emb_len / dims;
    if (n == 0 || scores_len < n) return;
    for (size_t i = 0; i < n; i++) scores[i] = orc_euclid(emb + i * dims, dims, q, dims);
}
/* simd.BatchNormalize — pkg/simd/simd.go:240-256. */
void orc_batch_normalize(float *vectors, size_t len, size_t n, size_t dims) {
    if (n == 0 || dims == 0 || len < n * dims) return;
    for (size_t i = 0; i < n; i++) orc_normalize_inplace(vectors + i * dims, dims);
}

/* ---------------------------------------------------------------- pkg/math/vector ------ */

/* vector.CosineSimilarity — pkg/math/vector/similarity.go:34-51: fp32 products, fp64 accumulators. */
double orc_vec_cosine64(const float *a, size_t na, const float *b, size_t nb) {
    if (na != nb || na == 0) return 0.0;
    double dot = 0.0, xa = 0.0, xb = 0.0;
    for (size_t i = 0; i < na; i++) {
        dot += (double)(float)(a[i] * b[i]);
        xa += (double)(float)(a[i] * a[i]);
        xb += (double)(float)(b[i] * b[i]);
    }
    if (xa == 0.0 || xb == 0.0) return 0.0;
    return dot / (sqrt(xa) * sqrt(xb));
}

/* vector.DotProduct — similarity.go:122-124 (float64 of simd.DotProduct). */
double orc_vec_dot(const float *a, size_t na, const float *b, size_t nb) {
    return (double)orc_dot(a, na, b, nb);
}

/* vector.EuclideanSimilarity — similarity.go:152-158: 1/(1+dist). */
double orc_vec_euclid_sim(const float *a, size_t na, const float *b, size_t nb) {
    if (na != nb || na == 0) return 0.0;
    float dist = orc_euclid(a, na, b, nb);
    return 1.0 / (1.0 + (double)dist);
}

/* vector.Normalize — similarity.go:197-210: zero vector -> zero vector; multiply by 1/n. */
void orc_vec_normalize(const float *v, size_t n, float *out) {
    float nrm = orc_norm(v, n);
    if (nrm == 0.0f) {
        memset(out, 0, n * sizeof(float));
        return;
    }
    float inv = 1.0f / nrm;
    for (size_t i = 0; i < n; i++) out[i] = v[i] * inv;
}

/* ---------------------------------------------------------------- pkg/gpu -------------- */

/* sqrt32 — pkg/gpu/gpu.go:1079-1089: ten Newton steps from z=x. */
static float orc_sqrt32(float x) {
    if (x <= 0.0f) return 0.0f;
    float z = x;
    for (int i = 0; i < 10; i++) z = (z + x / z) / 2.0f;
    return z;
}

/* cosineSimilarityFlat — pkg/gpu/gpu.go:2467-2484. */
float orc_cosine_flat(const float *a, size_t na, const float *b, size_t nb) {
    if (na != nb) return 0.0f;
    float dot = 0.0f, xa = 0.0f, xb = 0.0f;
    for (size_t i = 0; i < na; i++) {
        dot += a[i] * b[i];
        xa += a[i] * a[i];
        xb += b[i] * b[i];
    }
    if (xa == 0.0f || xb == 0.0f) return 0.0f;
    return dot / (orc_sqrt32(xa) * orc_sqrt32(xb));
}

/* partialSort — pkg/gpu/gpu.go:2507-2530 (swap-based selection, strict >). */
void orc_partial_sort(int64_t *indices, size_t n, const float *scores, size_t k) {
    if (k >= n) {
        for (size_t i = 0; i + 1 < n; i++)
            for (size_t j = i + 1; j < n; j++)
                if (scores[indices[j]] > scores[indices[i]]) {
                    int64_t t = indices[i];
                    indices[i] = indices[j];
                    indices[j] = t;
                }
        return;
    }
    for (size_t i = 0; i < k; i++) {
        size_t mx = i;
        for (size_t j = i + 1; j < n; j++)
            if (scores[indices[j]] > scores[indices[mx]]) mx = j;
        int64_t t = indices[i];
        indices[i] = indices[mx];
        indices[mx] = t;
    }
}

/* cuda_topk — pkg/gpu/cuda/cuda_bridge.go:327-375: forward scan, strict '>', so among equal
 * scores the lowest index wins and appears first.  Returns the clamped k. */
unsigned orc_topk_insertion(const float *scores, unsigned n, unsigned k, unsigned *out_idx,
                            float *out_scores) {
    if (k == 0 || n == 0) return 0;
    if (k > n) k = n;
    for (unsigned i = 0; i < k; i++) {
        out_scores[i] = -1e30f;
        out_idx[i] = 0;
    }
    for (unsigned i = 0; i < n; i++) {
        float s = scores[i];
        if (s > out_scores[k - 1]) {
            unsigned pos = k - 1;
            while (pos > 0 && s > out_scores[pos - 1]) {
                out_scores[pos] = out_scores[pos - 1];
                out_idx[pos] = out_idx[pos - 1];
                pos--;
            }
            out_scores[pos] = s;
            out_idx[pos] = i;
        }
    }
    return k;
}

/* ---------------------------------------------------------------- synthetic corpora ---- */

/* Counter-based generator shared bit-for-bit with the device (csrc/rowops.cu nk_fill kernel):
 * splitmix64 finaliser of (seed, element index) -> 24 random bits -> U[-1,1) on a 2^-23 grid
 * (every value exactly representable in fp32).  Mirrors the U[-1,1) corpora of the reference's
 * own benchmarks (pkg/simd/benchmark_test.go:14-22, pkg/search/hnsw_recall_test.go:37). */
static inline uint64_t orc_mix64(uint64_t z) {
    z ^= z >> 30;
    z *= 0xBF58476D1CE4E5B9ULL;
    z ^= z >> 27;
    z *= 0x94D049BB133111EBULL;
    z ^= z >> 31;
    return z;
}
static inline float orc_uniform_at(uint64_t seed, uint64_t elem) {
    uint64_t z = orc_mix64((seed + 1) * 0x9E3779B97F4A7C15ULL + elem * 0xD1B54A32D192ED03ULL);
    uint32_t m = (uint32_t)(z >> 40); /* 24 bits */
    return (float)m * (1.0f / 8388608.0f) - 1.0f;
}
void orc_fill_uniform(float *out, uint64_t n_rows, uint64_t dim, uint64_t seed, uint64_t row_base) {
#pragma omp parallel for schedule(static)
    for (int64_t r = 0; r < (int64_t)n_rows; r++)
        for (uint64_t j = 0; j < dim; j++)
            out[(uint64_t)r * dim + j] = orc_uniform_at(seed, ((uint64_t)r + row_base) * dim + j);
}
/* Same stream rounded to IEEE binary16 (round-to-nearest-even), returned as raw u16 bits. */
void orc_fill_uniform_f16(uint16_t *out, uint64_t n_rows, uint64_t dim, uint64_t seed, uint64_t row_base) {
#pragma omp parallel for schedule(static)
    for (int64_t r = 0; r < (int64_t)n_rows; r++)
        for (uint64_t j = 0; j < dim; j++) {
            _Float16 h = (_Float16)orc_uniform_at(seed, ((uint64_t)r + row_base) * dim + j);
            uint16_t bits;
            memcpy(&bits, &h, 2);
            out[(uint64_t)r * dim + j] = bits;
        }
}
void orc_f16_to_f32(const uint16_t *in, float *out, uint64_t n) {
    for (uint64_t i = 0; i < n; i++) {
        _Float16 h;
        memcpy(&h, &in[i], 2);
        out[i] = (float)h;
    }
}

/* ---------------------------------------------------------------- exact fp64 kNN ------- */

typedef struct {
    double score;
    uint32_t idx;
} orc_cand;

/* (score desc, row index asc) — the tie rule of the C boundary, cuda_bridge.go:356-371.
 * For Euclidean the caller passes score = -dist^2 so the same rule yields (distance asc, index asc). */
static inline int orc_better(double s, uint32_t i, const orc_cand *c) {
    return s > c->score || (s == c->score && i < c->idx);
}

static inline double orc_elem(const void *rows, int dtype, uint64_t off) {
    if (dtype == ORC_F16) {
        _Float16 h;
        memcpy(&h, (const uint16_t *)rows + off, 2);
        return (double)h;
    }
    return (double)((const float *)rows)[off];
}

/* Exact brute-force kNN: every product and sum in fp64 (products of fp32/fp16 inputs are exact in
 * fp64), bounded insertion top-k.  Score semantics follow what callers see:
 *   cosine    : dot/(|x||q|), 0 if either norm is 0     (simd.go:62-67, similarity.go:34-51)
 *   dot       : sum x*q                                   (simd.go:38-43)
 *   euclidean : ranked by distance ascending; out_score = sqrt(sum (x-q)^2)  (simd.go:83-88)
 * k is clamped to n (cuda_bridge.go:647-649).  out_idx/out_score are [Q x k_eff] row-major with
 * stride k (unclamped).  Returns k_eff. */
unsigned orc_knn_exact64(const void *rows, int dtype, uint64_t n, uint32_t dim, uint64_t row_base,
                         const float *queries, uint32_t Q, uint32_t k, int metric, uint32_t *out_idx,
                         double *out_score) {
    if (k == 0 || n == 0 || Q == 0) return 0;
    uint32_t ke = k > n ? (uint32_t)n : k;
#pragma omp parallel for schedule(dynamic, 1)
    for (int64_t qi = 0; qi < (int64_t)Q; qi++) {
        const float *q = queries + (uint64_t)qi * dim;
        orc_cand *top = (orc_cand *)malloc(sizeof(orc_cand) * ke);
        uint32_t cnt = 0;
        double qq = 0.0;
        for (uint32_t j = 0; j < dim; j++) qq += (double)q[j] * (double)q[j];
        for (uint64_t r = 0; r < n; r++) {
            double dot = 0.0, xx = 0.0, dd = 0.0;
            uint64_t off = r * dim;
            if (metric == ORC_EUCLIDEAN) {
                for (uint32_t j = 0; j < dim; j++) {
                    double diff = orc_elem(rows, dtype, off + j) - (double)q[j];
                    dd += diff * diff;
                }
            } else {
                for (uint32_t j = 0; j < dim; j++) {
                    double x = orc_elem(rows, dtype, off + j);
                    dot += x * (double)q[j];
                    xx += x * x;
                }
            }
            double s;
            if (metric == ORC_COSINE)
                s = (xx == 0.0 || qq == 0.0) ? 0.0 : dot / (sqrt(xx) * sqrt(qq));
            else if (metric == ORC_DOT)
                s = dot;
            else
                s = -dd;
            uint32_t gi = (uint32_t)(r + row_base);
            if (cnt < ke) {
                uint32_t pos = cnt++;
                while (pos > 0 && orc_better(s, gi, &top[pos - 1])) {
                    top[pos] = top[pos - 1];
                    pos--;
                }
                top[pos].score = s;
                top[pos].idx = gi;
            } else if (orc_better(s, gi, &top[ke - 1])) {
                uint32_t pos = ke - 1;
                while (pos > 0 && orc_better(s, gi, &top[pos - 1])) {
                    top[pos] = top[pos - 1];
                    pos--;
                }
                top[pos].score = s;
                top[pos].idx = gi;
            }
        }
        for (uint32_t i = 0; i < ke; i++) {
            out_idx[(uint64_t)qi * k + i] = top[i].idx;
            out_score[(uint64_t)qi * k + i] = metric == ORC_EUCLIDEAN ? sqrt(-top[i].score) : top[i].score;
        }
        free(top);
    }
    return ke;
}

/* All n scores of one query in fp64 (used by tests to classify boundary swaps: an index that
 * differs from the oracle's is acceptable only if its fp64 score is within fp32 summation noise
 * of the k-th score — SURVEY.md §8d "parity rule").  Euclidean returns the distance. */
void orc_scores_exact64(const void *rows, int dtype, uint64_t n, uint32_t dim, const float *q, int metric,
                        double *out) {
    double qq = 0.0;
    for (uint32_t j = 0; j < dim; j++) qq += (double)q[j] * (double)q[j];
#pragma omp parallel for schedule(static)
    for (int64_t r = 0; r < (int64_t)n; r++) {
        double dot = 0.0, xx = 0.0, dd = 0.0;
        uint64_t off = (uint64_t)r * dim;
        for (uint32_t j = 0; j < dim; j++) {
            double x = orc_elem(rows, dtype, off + j);
            double diff = x - (double)q[j];
            dot += x * (double)q[j];
            xx += x * x;
            dd += diff * diff;
        }
        if (metric == ORC_COSINE)
            out[r] = (xx == 0.0 || qq == 0.0) ? 0.0 : dot / (sqrt(xx) * sqrt(qq));
        else if (metric == ORC_DOT)
            out[r] = dot;
        else
            out[r] = sqrt(dd);
    }
}

int orc_num_threads(void) {
#ifdef _OPENMP
    return omp_get_max_threads();
#else
    return 1;
#endif
}

/* ======================================================================================================
 * k-means routing (pkg/gpu/kmeans.go) — SURVEY.md §8(f)4
 * ====================================================================================================== */

/* squaredEuclidean — kmeans.go:430-454: float32 differences, float64 squares in four interleaved sums. */
double orc_sq_euclid64(const float *a, const float *b, size_t n) {
    double s0 = 0.0, s1 = 0.0, s2 = 0.0, s3 = 0.0;
    size_t i = 0;
    for (; i + 4 <= n; i += 4) {
        double d0 = (double)(a[i] - b[i]), d1 = (double)(a[i + 1] - b[i + 1]);
        double d2 = (double)(a[i + 2] - b[i + 2]), d3 = (double)(a[i + 3] - b[i + 3]);
        s0 += d0 * d0; s1 += d1 * d1; s2 += d2 * d2; s3 += d3 * d3;
    }
    for (; i < n; i++) {
        double d = (double)(a[i] - b[i]);
        s0 += d * d;
    }
    return s0 + s1 + s2 + s3;
}

/* assignToCentroids — kmeans.go:458-489 (by_cosine = 0: nearest by squaredEuclidean, strict <) and
 * assignToCentroidsGPU — kmeans.go:491-546 (by_cosine = 1: highest cosineSimilarityFlat, strict >).
 * assign[] is updated in place; returns the number of assignments that changed. */
uint64_t orc_kmeans_assign(const float *rows, uint64_t n, uint32_t dim, const float *centroids, uint32_t k, int by_cosine,
                           int32_t *assign) {
    uint64_t changed = 0;
    for (uint64_t i = 0; i < n; i++) {
        const float *x = rows + i * dim;
        int32_t nearest = 0;
        if (by_cosine) {
            float best = -FLT_MAX;
            for (uint32_t c = 0; c < k; c++) {
                float sim = orc_cosine_flat(centroids + (size_t)c * dim, dim, x, dim);
                if (sim > best) { best = sim; nearest = (int32_t)c; }
            }
        } else {
            double best = DBL_MAX;
            for (uint32_t c = 0; c < k; c++) {
                double d = orc_sq_euclid64(x, centroids + (size_t)c * dim, dim);
                if (d < best) { best = d; nearest = (int32_t)c; }
            }
        }
        if (assign[i] != nearest) { assign[i] = nearest; changed++; }
    }
    return changed;
}

/* updateCentroidsWithBuffer — kmeans.go:585-618: float64 sums, mean rounded to float32, empty clusters keep
 * their previous position.  counts (k) may be NULL. */
void orc_kmeans_update(const float *rows, uint64_t n, uint32_t dim, const int32_t *assign, uint32_t k, float *centroids,
                       uint32_t *counts) {
    double *sums = (double *)calloc((size_t)k * dim, sizeof(double));
    uint64_t *cnt = (uint64_t *)calloc(k, sizeof(uint64_t));
    for (uint64_t i = 0; i < n; i++) {
        int32_t c = assign[i];
        if (c < 0 || (uint32_t)c >= k) continue;
        cnt[c]++;
        for (uint32_t d = 0; d < dim; d++) sums[(size_t)c * dim + d] += (double)rows[i * dim + d];
    }
    for (uint32_t c = 0; c < k; c++) {
        if (cnt[c] > 0)
            for (uint32_t d = 0; d < dim; d++) centroids[(size_t)c * dim + d] = (float)(sums[(size_t)c * dim + d] / (double)cnt[c]);
        if (counts) counts[c] = (uint32_t)cnt[c];
    }
    free(sums);
    free(cnt);
}
