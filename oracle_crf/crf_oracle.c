/* oracle_crf/crf_oracle.c -- TEST INFRASTRUCTURE ONLY: a plain-C restatement of the reference's SimpleCRF
 * (src/simple-crf.hpp:135-174, src/simple-crf.cpp:34-163), stateless: the caller (oracle_crf/crf.py) keeps the frames.
 *
 * Compiled with -ffp-contract=off; every multiply-add the reference's object code (g++ -O3 -mavx2 -mfma) fuses is an
 * explicit fmaf here, every other operation is rounded on its own.  expf / logf / sqrtf are glibc's.
 */
#include <math.h>
#include <stddef.h>
#include <stdint.h>

typedef struct {
    float y, x, r, g, b, a;
    uint16_t number;
    uint8_t is_active, is_updatable;
    uint32_t num_members;
} Cluster; /* fast-slic-common.h:10-23 */

typedef struct {
    float spatial_w, temporal_w, spatial_srgb, temporal_srgb, spatial_sxy, spatial_smooth_w, spatial_smooth_sxy;
} Params; /* simple-crf.h:11-19 */

/* -(((c1-c2)/s)^2 summed over r, g, b): the object code squares g, fuses r then b in */
static float neg_rgb(const Cluster* c1, const Cluster* c2, float s) {
    float dg = (c1->g - c2->g) / s, dr = (c1->r - c2->r) / s, db = (c1->b - c2->b) / s;
    return -fmaf(db, db, fmaf(dr, dr, dg * dg));
}

static float neg_xy(const Cluster* c1, const Cluster* c2, float s) {
    float dx = (c1->x - c2->x) / s, dy = (c1->y - c2->y) / s;
    return -fmaf(dx, dx, dy * dy);
}

/* simple-crf.hpp:149-174 (node_i != node_j) */
float orcl_crf_spatial_energy(const Cluster* c1, const Cluster* c2, const Params* p) {
    float exponent = fmaf(neg_rgb(c1, c2, p->spatial_srgb), 0.5f, neg_xy(c1, c2, p->spatial_sxy) * 0.5f);
    float smooth = neg_xy(c1, c2, p->spatial_smooth_sxy) * 0.5f;
    float e = expf(exponent);
    float es = expf(smooth);
    return fmaf(p->spatial_w, e, es * p->spatial_smooth_w);
}

/* simple-crf.hpp:135-147 (two different frames) */
float orcl_crf_temporal_energy(const Cluster* c1, const Cluster* c2, const Params* p) {
    return expf(neg_rgb(c1, c2, p->temporal_srgb) * 0.5f) * p->temporal_w;
}

/* simple-crf.cpp:34-55 */
void orcl_crf_unbiased(size_t C, size_t N, float* u) {
    float v = logf((float)C);
    for (size_t k = 0; k < C * N; k++) u[k] = v;
}

void orcl_crf_mask(size_t C, size_t N, const int32_t* classes, float confidence, float* u) {
    float lowest = 1.0f / (float)C;
    float active = fmaf(1.0f - lowest, confidence, lowest);
    float inactive = (1.0f - active) / (float)(C - 1);
    float au = -logf(active), iu = -logf(inactive);
    for (size_t k = 0; k < C * N; k++) u[k] = iu;
    for (size_t i = 0; i < N; i++) u[N * (size_t)classes[i] + i] = au;
}

void orcl_crf_proba(size_t n, const float* p, float* u) {
    for (size_t k = 0; k < n; k++) u[k] = -logf(p[k]);
}

/* simple-crf.cpp:57-59 */
void orcl_crf_reset(size_t n, const float* u, float* q) {
    for (size_t k = 0; k < n; k++) q[k] = expf(-u[k]);
}

static float ratio(uint32_t m_other, float m_i) { return sqrtf((float)m_other / m_i); }

/* One infer_once (simple-crf.cpp:62-151) over T frames in time order: q[t] (in) -> q_new[t] (out).  msg and e are
 * scratch float[C*N]. */
static void infer_once(int T, size_t C, size_t N, const Cluster* const* cl, const int32_t* const* off,
                       const int32_t* const* nbr, const float* const* unary, float* const* q, float* const* q_new,
                       const Params* p, float* msg, float* sums) {
    for (int t = 0; t < T; t++) {
        const Cluster* c = cl[t];
        for (size_t cls = 0; cls < C; cls++) {
            for (size_t i = 0; i < N; i++) {
                int mi_int = (int)c[i].num_members;
                if (mi_int <= 0) mi_int = 1;
                float mi = (float)mi_int;
                float m = 0;
                for (int32_t k = off[t][i]; k < off[t][i + 1]; k++) {
                    int j = nbr[t][k];
                    float e = (size_t)j == i ? 0.0f : orcl_crf_spatial_energy(&c[j], &c[i], p);
                    m = fmaf(e * q[t][N * cls + j], ratio(c[j].num_members, mi), m);
                }
                if (t > 0) {
                    const Cluster* o = &cl[t - 1][i];
                    m = fmaf(orcl_crf_temporal_energy(&c[i], o, p) * q[t - 1][N * cls + i], ratio(o->num_members, mi), m);
                }
                if (t < T - 1) {
                    const Cluster* o = &cl[t + 1][i];
                    m = fmaf(orcl_crf_temporal_energy(&c[i], o, p) * q[t + 1][N * cls + i], ratio(o->num_members, mi), m);
                }
                msg[cls * N + i] = m;
            }
        }
        float* e = q_new[t];
        for (size_t cls = 0; cls < C; cls++) {
            for (size_t i = 0; i < N; i++) {
                float acc = 0;
                for (size_t o = 0; o < C; o++) {
                    if (o == cls) continue;
                    acc = fmaf(1.0f, msg[o * N + i], acc); /* compat_by_class[o] == 1 */
                }
                e[cls * N + i] = expf(-(unary[t][cls * N + i] + acc));
            }
        }
        for (size_t i = 0; i < N; i++) sums[i] = 0.0f;
        for (size_t cls = 0; cls < C; cls++)
            for (size_t i = 0; i < N; i++) sums[i] += e[N * cls + i];
        for (size_t i = 0; i < N; i++) sums[i] = ((double)sums[i] < 1e-5) ? 1e-5f : sums[i];
        for (size_t cls = 0; cls < C; cls++)
            for (size_t i = 0; i < N; i++) e[N * cls + i] /= sums[i];
    }
}

/* max_iter infer_once calls; q[t] is updated in place (work: 2 * T * C * N + N floats of scratch) */
void orcl_crf_inference(int T, size_t C, size_t N, const Cluster* const* cl, const int32_t* const* off,
                        const int32_t* const* nbr, const float* const* unary, float* const* q, const Params* p,
                        long long max_iter, float* work) {
    float* qn[4096];
    for (int t = 0; t < T; t++) qn[t] = work + (size_t)t * C * N;
    float* msg = work + (size_t)T * C * N;
    float* sums = msg + C * N;
    for (long long it = 0; it < max_iter; it++) {
        infer_once(T, C, N, cl, off, nbr, unary, q, qn, p, msg, sums);
        for (int t = 0; t < T; t++)
            for (size_t k = 0; k < C * N; k++) q[t][k] = qn[t][k];
    }
}

/* glibc's expf over the bit patterns first .. first + n - 1 */
void orcl_expf_range(uint32_t first, long long n, float* out) {
    for (long long i = 0; i < n; i++) {
        union { uint32_t u; float f; } v;
        v.u = first + (uint32_t)i;
        out[i] = expf(v.f);
    }
}

/* glibc's logf over the bit patterns first .. first + n - 1 */
void orcl_logf_range(uint32_t first, long long n, float* out) {
    for (long long i = 0; i < n; i++) {
        union { uint32_t u; float f; } v;
        v.u = first + (uint32_t)i;
        out[i] = logf(v.f);
    }
}
