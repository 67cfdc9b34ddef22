/*
 * oracle_lsc/lsc_oracle.c -- TEST INFRASTRUCTURE ONLY.
 *
 * The plain-C restatement of the reference's ContextLSC (src/lsc.cpp, lsc.h; linear spectral clustering) driven with
 * num_threads = 1, the only thread count whose result is defined (DESIGN.md section 4.9).  BaseContext::iterate
 * (context.cpp:109-197), the scheduler of assign() (:200-243), the integer update (:302-387) and connectivity
 * enforcement are the Manhattan restatement's own code: this file includes oracle/slic_oracle.c and adds the three hooks
 * LSC overrides (before_iteration, assign_clusters, after_update).  Pinned to the compiled reference by
 * tests/test_lsc_cpu.py against tests/golden/lsc_reference_digests.npz (tests/golden/make_lsc_golden.py).
 *
 * Each float operation is written the way the reference's object code (g++ -O3 -mfma, oracle/Makefile) evaluates it.
 * This file is ISO C, so nothing is contracted behind our back: the steps GCC fuses there are fmaf here.
 */
#define _GNU_SOURCE /* sincos */
#include "../oracle/slic_oracle.c"

#include <float.h>

#define NFEAT 10

/* lsc.cpp:25-28 and :69-101.  The reference calls glibc's double sin / cos on a float angle (GCC merges each pair into
 * one sincos call); the colour tables round the cosine to float first, the others multiply in double. */
typedef struct {
    float Lc[256], Ls[256], Cc[256], Cs[256];
    float *Wc, *Ws, *Hc, *Hs;
} LscTables;

static void lsc_tables(int H, int W, int S, float compactness, LscTables* t) {
    const float PI = (float)3.1415926;
    const float halfPI = PI / 2;
    const float ratio = compactness / 100.0f;
    const float C_color = 20.0f; /* lsc.h:8 */
    const float C_spatial = C_color * ratio;
    double s, c;
    for (int X = 0; X < 256; X++) { /* :78-83 */
        float theta = halfPI * ((float)X / 255.0f);
        sincos((double)theta, &s, &c);
        float cosine = (float)c, sine = (float)s;
        t->Cc[X] = C_color * cosine * 2.55f;
        t->Cs[X] = C_color * sine * 2.55f;
    }
    for (int X = 0; X < 256; X++) { /* :85-89 */
        float theta = halfPI * ((float)X / 255.0f);
        sincos((double)theta, &s, &c);
        t->Lc[X] = (float)((double)C_color * c);
        t->Ls[X] = (float)((double)C_color * s);
    }
    t->Hc = (float*)malloc(sizeof(float) * (size_t)H);
    t->Hs = (float*)malloc(sizeof(float) * (size_t)H);
    t->Wc = (float*)malloc(sizeof(float) * (size_t)W);
    t->Ws = (float*)malloc(sizeof(float) * (size_t)W);
    const float step = halfPI / (float)S;
    for (int i = 0; i < H; i++) { /* :91-95 */
        float theta = (float)i * step;
        sincos((double)theta, &s, &c);
        t->Hc[i] = (float)((double)C_spatial * c);
        t->Hs[i] = (float)((double)C_spatial * s);
    }
    for (int i = 0; i < W; i++) { /* :97-101 */
        float theta = (float)i * step;
        sincos((double)theta, &s, &c);
        t->Wc[i] = (float)((double)C_spatial * c);
        t->Ws[i] = (float)((double)C_spatial * s);
    }
}

/* map_image_into_feature_space, lsc.cpp:22-163: the ten raw features per pixel (:103-135), their means -- one serial
 * float sum over all pixels per feature, divided by the pixel count (:138-150) --, the weight
 * w = sum_f mean_f * feat_f as a fused chain from 0 (:151-160), and every feature divided by its pixel's weight (:161,
 * normalize_features :309-316).  feat is [10][H*W]. */
static void map_image(int H, int W, int S, float compactness, const uint8_t* quad, float* feat, float* weights,
                      float* means) {
    LscTables t;
    lsc_tables(H, W, S, compactness, &t);
    const long len = (long)H * W;
    for (int i = 0; i < H; i++)
        for (int j = 0; j < W; j++) {
            long p = (long)i * W + j;
            int L = quad[4 * p], A = quad[4 * p + 1], B = quad[4 * p + 2];
            feat[0 * len + p] = t.Lc[L];
            feat[1 * len + p] = t.Ls[L];
            feat[2 * len + p] = t.Cc[A];
            feat[3 * len + p] = t.Cs[A];
            feat[4 * len + p] = t.Cc[B];
            feat[5 * len + p] = t.Cs[B];
            feat[6 * len + p] = t.Wc[j];
            feat[7 * len + p] = t.Ws[j];
            feat[8 * len + p] = t.Hc[i];
            feat[9 * len + p] = t.Hs[i];
        }
    for (int f = 0; f < NFEAT; f++) {
        float sum = 0;
        for (long p = 0; p < len; p++) sum = sum + feat[f * len + p];
        means[f] = sum / (float)len;
    }
    for (long p = 0; p < len; p++) {
        float w = 0;
        for (int f = 0; f < NFEAT; f++) w = fmaf(means[f], feat[f * len + p], w);
        weights[p] = w;
    }
    for (long p = 0; p < len; p++)
        for (int f = 0; f < NFEAT; f++) feat[f * len + p] = feat[f * len + p] / weights[p];
    free(t.Hc); free(t.Hs); free(t.Wc); free(t.Ws);
}

/* map_centroids_into_feature_space, lsc.cpp:165-195: the mean normalised feature over the clamped (2 (S/4) + 1)^2
 * window around each (unclamped, truncated) centre, summed in raster order; an empty window gives 0/0.  cf is [K][10]. */
static void map_centroids(int H, int W, int K, int S, const OrcCluster* clusters, const float* feat, float* cf) {
    const long len = (long)H * W;
    for (int k = 0; k < K; k++) {
        int cy = (int)clusters[k].y, cx = (int)clusters[k].x;
        int y_lo = cy - S / 4 > 0 ? cy - S / 4 : 0, y_hi = cy + S / 4 + 1 < H ? cy + S / 4 + 1 : H;
        int x_lo = cx - S / 4 > 0 ? cx - S / 4 : 0, x_hi = cx + S / 4 + 1 < W ? cx + S / 4 + 1 : W;
        float acc[NFEAT] = {0}, wsum = 0.0f;
        for (int i = y_lo; i < y_hi; i++)
            for (int j = x_lo; j < x_hi; j++) {
                long p = (long)i * W + j;
                for (int f = 0; f < NFEAT; f++) acc[f] = acc[f] + feat[f * len + p];
                wsum = wsum + 1.0f;
            }
        for (int f = 0; f < NFEAT; f++) cf[k * NFEAT + f] = acc[f] / wsum;
    }
}

/* assign() (context.cpp:200-243) with ContextLSC::assign_clusters (lsc.cpp:197-224): clusters clamped into the image
 * and bucketed per T x T cell, cells visited in four phases; the window is the clamped (2S+1)^2 square around the
 * truncated centre; d = sum_f (feat_f - centroid_f)^2 as the fused chain fma(diff, diff, d) from 0, kept only when
 * strictly below the running minimum (FLT_MAX at first: NaN and +inf never win). */
static void assign_pass_lsc(int H, int W, int K, int S, OrcCluster* clusters, const float* feat, const float* cf,
                            uint16_t* assignment, float* min_dists, int stride, int rem) {
    const long len = (long)H * W;
    for (long p = 0; p < len; p++) min_dists[p] = FLT_MAX;
    for (int k = 0; k < K; k++) { /* context.cpp:209-212 */
        float x = clusters[k].x, y = clusters[k].y;
        clusters[k].x = x < 0 ? 0 : (x > (float)(W - 1) ? (float)(W - 1) : x);
        clusters[k].y = y < 0 ? 0 : (y > (float)(H - 1) ? (float)(H - 1) : y);
    }
    int T = 2 * S + 32;
    int cell_W = ceil_int(W, T), cell_H = ceil_int(H, T), ncell = cell_W * cell_H;
    int* start = (int*)calloc((size_t)ncell + 1, sizeof(int));
    int* items = (int*)malloc(sizeof(int) * (size_t)K);
    for (int k = 0; k < K; k++)
        if (clusters[k].is_active) start[cell_W * ((int)clusters[k].y / T) + ((int)clusters[k].x / T) + 1]++;
    for (int c = 0; c < ncell; c++) start[c + 1] += start[c];
    int* fill = (int*)malloc(sizeof(int) * (size_t)ncell);
    memcpy(fill, start, sizeof(int) * (size_t)ncell);
    for (int k = 0; k < K; k++)
        if (clusters[k].is_active) items[fill[cell_W * ((int)clusters[k].y / T) + ((int)clusters[k].x / T)]++] = k;
    for (int phase = 0; phase < 4; phase++)
        for (int ci = phase / 2; ci < cell_H; ci += 2)
            for (int cj = phase % 2; cj < cell_W; cj += 2) {
                int cell = ci * cell_W + cj;
                for (int t = start[cell]; t < start[cell + 1]; t++) {
                    const OrcCluster* c = &clusters[items[t]];
                    int cy = (int)c->y, cx = (int)c->x;
                    uint16_t no = c->number;
                    int y_lo = cy - S > 0 ? cy - S : 0, y_hi = cy + S + 1 < H ? cy + S + 1 : H;
                    int x_lo = cx - S > 0 ? cx - S : 0, x_hi = cx + S + 1 < W ? cx + S + 1 : W;
                    for (int i = y_lo; i < y_hi; i++) {
                        if (i % stride != rem) continue;
                        for (int j = x_lo; j < x_hi; j++) {
                            long p = (long)i * W + j;
                            float d = 0;
                            for (int f = 0; f < NFEAT; f++) {
                                float diff = feat[f * len + p] - cf[(long)no * NFEAT + f];
                                d = fmaf(diff, diff, d);
                            }
                            if (min_dists[p] > d) {
                                min_dists[p] = d;
                                assignment[p] = no;
                            }
                        }
                    }
                }
            }
    free(start); free(items); free(fill);
}

/* ContextLSC::after_update (lsc.cpp:226-307) with one thread: per cluster, the raster-order sums over the pass's rows of
 * w * feat_f (fused into the running sum) and of w; an updatable cluster's centroid becomes (0 + sum_f) / (0 + sum_w)
 * -- 0/0 = NaN for a cluster without pixels --, any other adds its old value and 1 to the sums. */
static void after_update_lsc(int H, int W, int K, const OrcCluster* clusters, const float* feat, const float* weights,
                             const uint16_t* assignment, float* cf, int stride, int rem) {
    const long len = (long)H * W;
    float* lf = (float*)calloc((size_t)K * NFEAT, sizeof(float));
    float* lw = (float*)calloc((size_t)K, sizeof(float));
    for (int i = rem; i < H; i += stride)
        for (int j = 0; j < W; j++) {
            long p = (long)i * W + j;
            uint16_t c = assignment[p];
            if (c == 0xFFFF) continue;
            float w = weights[p];
            for (int f = 0; f < NFEAT; f++) lf[(long)c * NFEAT + f] = fmaf(w, feat[f * len + p], lf[(long)c * NFEAT + f]);
            lw[c] = lw[c] + w;
        }
    for (int k = 0; k < K; k++) {
        int up = clusters[k].is_updatable != 0;
        float wsum = (up ? 0.0f : 1.0f) + lw[k];
        for (int f = 0; f < NFEAT; f++) {
            float base = up ? 0.0f : cf[k * NFEAT + f];
            cf[k * NFEAT + f] = (base + lf[(long)k * NFEAT + f]) / wsum;
        }
    }
    free(lf); free(lw);
}

/* BaseContext<float>::iterate (context.cpp:109-197) on a ContextLSC.  The stage outputs may be NULL:
 * means_out float[10], weights_out float[H*W], cinit_out / cfinal_out float[K][10] (centroid features after
 * before_iteration / at the end), precca_out u16[H*W]. */
void orcl_iterate_lsc(int H, int W, int K, const uint8_t* image, OrcCluster* clusters, uint16_t* out, int max_iter,
                      float compactness, float min_size_factor, int stride, int convert_to_lab, uint16_t* precca_out,
                      float* means_out, float* weights_out, float* cinit_out, float* cfinal_out) {
    if (H <= 0 || W <= 0 || K <= 0) return;
    int S = (int16_t)sqrt((double)(H * W / K)); /* context.h:60 */
    long N = (long)H * W;
    uint8_t* quad = (uint8_t*)malloc((size_t)N * 4);
    uint16_t* assignment = (uint16_t*)malloc(sizeof(uint16_t) * (size_t)N);
    float* min_dists = (float*)malloc(sizeof(float) * (size_t)N);
    float* feat = (float*)malloc(sizeof(float) * (size_t)N * NFEAT);
    float* weights = (float*)malloc(sizeof(float) * (size_t)N);
    float* cf = (float*)malloc(sizeof(float) * (size_t)K * NFEAT);
    float means[NFEAT];
    orc_rgb_to_quad(image, H, W, convert_to_lab, quad);
    for (int k = 0; k < K; k++) {
        int y = clampi((int)clusters[k].y, 0, H - 1), x = clampi((int)clusters[k].x, 0, W - 1);
        clusters[k].r = quad[4 * ((long)y * W + x)];
        clusters[k].g = quad[4 * ((long)y * W + x) + 1];
        clusters[k].b = quad[4 * ((long)y * W + x) + 2];
    }
    for (long p = 0; p < N; p++) assignment[p] = 0xFFFF;
    map_image(H, W, S, compactness, quad, feat, weights, means); /* before_iteration, lsc.cpp:12-15 */
    map_centroids(H, W, K, S, clusters, feat, cf);
    if (means_out) memcpy(means_out, means, sizeof(means));
    if (weights_out) memcpy(weights_out, weights, sizeof(float) * (size_t)N);
    if (cinit_out) memcpy(cinit_out, cf, sizeof(float) * (size_t)K * NFEAT);
    for (int k = 0; k < K; k++) clusters[k].is_updatable = 2; /* preemptive.h:59-67 */
    int rem = 0;
    for (int it = 0; it < max_iter; it++) {
        assign_pass_lsc(H, W, K, S, clusters, feat, cf, assignment, min_dists, stride, rem);
        update_pass(H, W, K, clusters, quad, assignment, stride, rem);
        after_update_lsc(H, W, K, clusters, feat, weights, assignment, cf, stride, rem);
        rem = (rem + 1) % stride;
    }
    for (int k = 0; k < K; k++) clusters[k].is_active = 1;
    assign_pass_lsc(H, W, K, S, clusters, feat, cf, assignment, min_dists, 1, 0);
    if (cfinal_out) memcpy(cfinal_out, cf, sizeof(float) * (size_t)K * NFEAT);
    if (precca_out) memcpy(precca_out, assignment, sizeof(uint16_t) * (size_t)N);
    memcpy(out, assignment, sizeof(uint16_t) * (size_t)N);
    orc_enforce_connectivity(out, H, W, K, (int)round((double)(S * S) * (double)min_size_factor));
    free(quad); free(assignment); free(min_dists); free(feat); free(weights); free(cf);
}
