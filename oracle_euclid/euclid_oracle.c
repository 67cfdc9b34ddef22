/*
 * oracle_euclid/euclid_oracle.c -- TEST INFRASTRUCTURE ONLY.
 *
 * The plain-C restatement of the reference with manhattan_spatial_dist = false (context.h:35): the Euclidean branch
 * of BaseContext::set_spatial_patch (context.cpp:34-38) for the u16 contexts (Slic / SlicAvx2, also with
 * `preemptive`) and ContextRealDist, and assign_clusters_proto<false> of ContextRealDistNoQ (context.cpp:462-496).
 * Everything the flag does not touch -- Lab conversion, seeding, the scheduler, the update, PreemptiveGrid,
 * connectivity enforcement -- is the Manhattan restatement's own code: this file includes oracle/slic_oracle.c and
 * only replaces the assign passes.  Pinned to the compiled reference by tests/test_euclidean_cpu.py against
 * tests/golden/euclid_reference_digests.npz (tests/golden/make_euclid_golden.py).
 */
#include "../oracle/slic_oracle.c"

/* The u16 patch, context.cpp:34-38 literally: (u16)(coef * hypotf(di, dj)) for the signed offsets di, dj in [-S, S],
 * stored at [(di + S) * (2S + 1) + (dj + S)]. */
static uint16_t* euclid_patch(int S, float coef) {
    int n = 2 * S + 1;
    uint16_t* patch = (uint16_t*)malloc(sizeof(uint16_t) * (size_t)n * (size_t)n);
    for (int i = 0; i < n; i++)
        for (int j = 0; j < n; j++) patch[(long)i * n + j] = (uint16_t)(coef * hypotf((float)(i - S), (float)(j - S)));
    return patch;
}

static float spatial_coef(int S, float compactness, int color_shift) { /* context.cpp:25-26 */
    float coef = 1.0f / ((float)S / compactness);
    coef *= (float)(1 << color_shift);
    return coef;
}

/* The scheduler of context.cpp:200-243 as assign_pass_bucketed has it: clusters clamped into the image, bucketed per
 * T x T cell (ascending k inside a cell), cells visited in four phases.  Returns start[ncell + 1] / items[K]. */
static void bucket_clusters(int H, int W, int K, int S, OrcCluster* clusters, int* cell_W_out, int* cell_H_out,
                            int** start_out, int** items_out) {
    for (int k = 0; k < K; k++) {
        float x = clusters[k].x, y = clusters[k].y;
        clusters[k].x = x < 0 ? 0 : (x > (float)(W - 1) ? (float)(W - 1) : x);
        clusters[k].y = y < 0 ? 0 : (y > (float)(H - 1) ? (float)(H - 1) : y);
    }
    int T = 2 * S + 32;
    int cell_W = ceil_int(W, T), cell_H = ceil_int(H, T);
    int ncell = cell_W * cell_H;
    int* start = (int*)calloc((size_t)ncell + 1, sizeof(int));
    int* items = (int*)malloc(sizeof(int) * (size_t)(K > 0 ? K : 1));
    for (int k = 0; k < K; k++) {
        if (!clusters[k].is_active) continue;
        start[cell_W * ((int)clusters[k].y / T) + ((int)clusters[k].x / T) + 1]++;
    }
    for (int c = 0; c < ncell; c++) start[c + 1] += start[c];
    int* fill = (int*)malloc(sizeof(int) * (size_t)(ncell > 0 ? ncell : 1));
    memcpy(fill, start, sizeof(int) * (size_t)ncell);
    for (int k = 0; k < K; k++) {
        if (!clusters[k].is_active) continue;
        items[fill[cell_W * ((int)clusters[k].y / T) + ((int)clusters[k].x / T)]++] = k;
    }
    free(fill);
    *cell_W_out = cell_W; *cell_H_out = cell_H; *start_out = start; *items_out = items;
}

/* assign with the u16 Euclidean patch (context.cpp:259-298); strict '>' against min_dists, first visitor wins ties */
static void assign_pass_euclid(int H, int W, int K, int S, OrcCluster* clusters, const uint8_t* quad, const uint16_t* patch,
                               uint16_t* assignment, uint16_t* min_dists, int stride, int rem) {
    for (long p = 0; p < (long)H * W; p++) min_dists[p] = 0xFFFF;
    int cell_W, cell_H, *start, *items;
    bucket_clusters(H, W, K, S, clusters, &cell_W, &cell_H, &start, &items);
    const int n = 2 * S + 1;
    for (int phase = 0; phase < 4; phase++)
        for (int ci = phase / 2; ci < cell_H; ci += 2)
            for (int cj = phase % 2; cj < cell_W; cj += 2) {
                int cell = ci * cell_W + cj;
                for (int t = start[cell]; t < start[cell + 1]; t++) {
                    int k = items[t];
                    int16_t cy = (int16_t)clusters[k].y, cx = (int16_t)clusters[k].x;
                    int16_t cr = (int16_t)clusters[k].r, cg = (int16_t)clusters[k].g, cb = (int16_t)clusters[k].b;
                    int i0 = cy - S < 0 ? 0 : cy - S, i1 = cy + S >= H ? H - 1 : cy + S;
                    int j0 = cx - S < 0 ? 0 : cx - S, j1 = cx + S >= W ? W - 1 : cx + S;
                    for (int i = i0; i <= i1; i++) {
                        if (i % stride != rem) continue;
                        const long prow = (long)(i - cy + S) * n + S;
                        for (int j = j0; j <= j1; j++) {
                            long p = (long)i * W + j;
                            int r = quad[4 * p], g = quad[4 * p + 1], b = quad[4 * p + 2];
                            uint16_t d = (uint16_t)(abs(r - cr) + abs(g - cg) + abs(b - cb) + patch[prow + (j - cx)]);
                            if (min_dists[p] > d) {
                                min_dists[p] = d;
                                assignment[p] = clusters[k].number;
                            }
                        }
                    }
                }
            }
    free(start);
    free(items);
}

/* orc_iterate_preemptive (context.cpp:109-197, preemptive.h) with the Euclidean assign */
void orce_iterate_preemptive(int H, int W, int K, const uint8_t* image, OrcCluster* clusters, uint16_t* out, int max_iter,
                             float compactness, float min_size_factor, int stride, int convert_to_lab, int preemptive,
                             float preemptive_thres, uint8_t* quad_out, uint16_t* precca_out) {
    if (H <= 0 || W <= 0 || K <= 0) return;
    int S = (int16_t)sqrt((double)(H * W / K)); /* context.h:60 */
    long N = (long)H * W;
    uint8_t* quad = (uint8_t*)malloc((size_t)N * 4);
    uint16_t* assignment = (uint16_t*)malloc(sizeof(uint16_t) * (size_t)N);
    uint16_t* min_dists = (uint16_t*)malloc(sizeof(uint16_t) * (size_t)N);
    int color_shift = convert_to_lab ? OUTPUT_SHIFT : 0;
    orc_rgb_to_quad(image, H, W, convert_to_lab, quad);
    for (int k = 0; k < K; k++) {
        int y = clampi((int)clusters[k].y, 0, H - 1), x = clampi((int)clusters[k].x, 0, W - 1);
        clusters[k].r = quad[4 * ((long)y * W + x)];
        clusters[k].g = quad[4 * ((long)y * W + x) + 1];
        clusters[k].b = quad[4 * ((long)y * W + x) + 2];
    }
    for (long p = 0; p < N; p++) assignment[p] = 0xFFFF;
    uint16_t* patch = euclid_patch(S, spatial_coef(S, compactness, color_shift));
    for (int k = 0; k < K; k++) clusters[k].is_updatable = 2;
    int all_active = 1;
    int* active_grid = NULL;
    float* old_yx = NULL;
    if (preemptive && S > 0) {
        active_grid = (int*)calloc((size_t)ceil_int(W, 2 * S) * ceil_int(H, 2 * S), sizeof(int));
        old_yx = (float*)malloc(sizeof(float) * 2 * (size_t)K);
    }
    int rem = 0;
    for (int it = 0; it < max_iter; it++) {
        assign_pass_euclid(H, W, K, S, clusters, quad, patch, assignment, min_dists, stride, rem);
        if (active_grid) {
            for (int k = 0; k < K; k++) {
                old_yx[2 * k] = clusters[k].y;
                old_yx[2 * k + 1] = clusters[k].x;
            }
            update_pass_masked(H, W, K, clusters, quad, assignment, stride, rem, all_active ? NULL : active_grid, 2 * S,
                               ceil_int(W, 2 * S));
            all_active = set_new_clusters(H, W, K, S, preemptive_thres, clusters, old_yx, active_grid);
        } else {
            update_pass(H, W, K, clusters, quad, assignment, stride, rem);
        }
        rem = (rem + 1) % stride;
    }
    free(active_grid);
    free(old_yx);
    for (int k = 0; k < K; k++) clusters[k].is_active = 1;
    assign_pass_euclid(H, W, K, S, clusters, quad, patch, assignment, min_dists, 1, 0);
    if (quad_out) memcpy(quad_out, quad, (size_t)N * 4);
    if (precca_out) memcpy(precca_out, assignment, sizeof(uint16_t) * (size_t)N);
    memcpy(out, assignment, sizeof(uint16_t) * (size_t)N);
    orc_enforce_connectivity(out, H, W, K, (int)round((double)(S * S) * (double)min_size_factor));
    free(quad); free(assignment); free(min_dists); free(patch);
}

/* float-distance contexts with manhattan_spatial_dist = false:
 *   variant 0  ContextRealDist: patch = coef * hypotf(di, dj), untruncated (context.cpp:34-38); d = patch + colour SAD
 *   variant 1  ContextRealDistL2 ignores the flag (:435-445): the Manhattan restatement's assign_pass_real
 *   variant 2  ContextRealDistNoQ, assign_clusters_proto<false> (:462-496): dr*dr + dg*dg + db*db + dx*dx + dy*dy, which
 *              the reference's object code (GCC, -mfma) evaluates as fma(dx, dx, fma(db, db, fma(dr, dr, dg*dg))) + dy*dy
 *              with dy*dy hoisted out of the row loop.  This file is ISO C (no contraction): the fused steps are fmaf. */
static void assign_pass_real_euclid(int variant, int H, int W, int K, int S, OrcCluster* clusters, const uint8_t* quad,
                                    float coef, uint16_t* assignment, float* min_dists, int stride, int rem) {
    for (long p = 0; p < (long)H * W; p++) min_dists[p] = 3.402823466e+38f;
    int cell_W, cell_H, *start, *items;
    bucket_clusters(H, W, K, S, clusters, &cell_W, &cell_H, &start, &items);
    for (int phase = 0; phase < 4; phase++)
        for (int ci = phase / 2; ci < cell_H; ci += 2)
            for (int cj = phase % 2; cj < cell_W; cj += 2) {
                int cell = ci * cell_W + cj;
                for (int t = start[cell]; t < start[cell + 1]; t++) {
                    const OrcCluster* c = &clusters[items[t]];
                    int i0, i1, j0, j1;
                    int16_t cy = (int16_t)c->y, cx = (int16_t)c->x;
                    int16_t cr = (int16_t)c->r, cg = (int16_t)c->g, cb = (int16_t)c->b;
                    if (variant == 2) { /* :472-473 */
                        i0 = (int)(c->y - (float)S); if (i0 < 0) i0 = 0;
                        i1 = (int)(c->y + (float)S + 1.0f); if (i1 > H) i1 = H;
                        j0 = (int)(c->x - (float)S); if (j0 < 0) j0 = 0;
                        j1 = (int)(c->x + (float)S + 1.0f); if (j1 > W) j1 = W;
                        i1--; j1--;
                    } else {
                        i0 = cy - S < 0 ? 0 : cy - S; i1 = cy + S >= H ? H - 1 : cy + S;
                        j0 = cx - S < 0 ? 0 : cx - S; j1 = cx + S >= W ? W - 1 : cx + S;
                    }
                    for (int i = i0; i <= i1; i++) {
                        if (i % stride != rem) continue;
                        for (int j = j0; j <= j1; j++) {
                            long p = (long)i * W + j;
                            int r = quad[4 * p], g = quad[4 * p + 1], b = quad[4 * p + 2];
                            float d;
                            if (variant == 0) {
                                float patch = coef * hypotf((float)(i - cy), (float)(j - cx));
                                d = patch + (float)(abs(r - cr) + abs(g - cg) + abs(b - cb));
                            } else {
                                float dr = (float)r - c->r, dg = (float)g - c->g, db = (float)b - c->b;
                                float dy = coef * ((float)i - c->y), dx = coef * ((float)j - c->x);
                                d = fmaf(dx, dx, fmaf(db, db, fmaf(dr, dr, dg * dg))) + dy * dy;
                            }
                            if (min_dists[p] > d) {
                                min_dists[p] = d;
                                assignment[p] = c->number;
                            }
                        }
                    }
                }
            }
    free(start);
    free(items);
}

/* orc_iterate_real (context.cpp:109-197 with the float contexts) with manhattan_spatial_dist = false */
void orce_iterate_real(int variant, int H, int W, int K, const uint8_t* image, OrcCluster* clusters, uint16_t* out,
                       int max_iter, float compactness, float min_size_factor, int stride, int convert_to_lab,
                       uint16_t* precca_out) {
    if (variant == 1) { /* the flag does not reach ContextRealDistL2 */
        orc_iterate_real(variant, H, W, K, image, clusters, out, max_iter, compactness, min_size_factor, stride,
                         convert_to_lab, precca_out);
        return;
    }
    if (H <= 0 || W <= 0 || K <= 0) return;
    int S = (int16_t)sqrt((double)(H * W / K));
    long N = (long)H * W;
    uint8_t* quad = (uint8_t*)malloc((size_t)N * 4);
    uint16_t* assignment = (uint16_t*)malloc(sizeof(uint16_t) * (size_t)N);
    float* min_dists = (float*)malloc(sizeof(float) * (size_t)N);
    orc_rgb_to_quad(image, H, W, convert_to_lab, quad);
    for (int k = 0; k < K; k++) {
        int y = clampi((int)clusters[k].y, 0, H - 1), x = clampi((int)clusters[k].x, 0, W - 1);
        clusters[k].r = quad[4 * ((long)y * W + x)];
        clusters[k].g = quad[4 * ((long)y * W + x) + 1];
        clusters[k].b = quad[4 * ((long)y * W + x) + 2];
    }
    for (long p = 0; p < N; p++) assignment[p] = 0xFFFF;
    float coef = spatial_coef(S, compactness, convert_to_lab ? OUTPUT_SHIFT : 0);
    for (int k = 0; k < K; k++) clusters[k].is_updatable = 2;
    int rem = 0;
    for (int it = 0; it < max_iter; it++) {
        assign_pass_real_euclid(variant, H, W, K, S, clusters, quad, coef, assignment, min_dists, stride, rem);
        update_pass_real(variant, H, W, K, clusters, quad, assignment, stride, rem);
        rem = (rem + 1) % stride;
    }
    for (int k = 0; k < K; k++) clusters[k].is_active = 1;
    assign_pass_real_euclid(variant, H, W, K, S, clusters, quad, coef, assignment, min_dists, 1, 0);
    if (precca_out) memcpy(precca_out, assignment, sizeof(uint16_t) * (size_t)N);
    memcpy(out, assignment, sizeof(uint16_t) * (size_t)N);
    orc_enforce_connectivity(out, H, W, K, (int)round((double)(S * S) * (double)min_size_factor));
    free(quad); free(assignment); free(min_dists);
}

/* The CUDA kernels do not call hypotf (CUDA's is not correctly rounded): they round the exact integer square sum's
 * square root themselves (euclid_dist, fast_slic_b200/csrc/assign.cuh) -- a float square root while the sum fits
 * 24 bits, a double one rounded to float beyond.  Returns how many offsets lo <= a, b <= hi this libm's hypotf
 * disagrees with that on. */
long orce_hypotf_mismatches(int lo, int hi) {
    long bad = 0;
    for (int a = lo; a <= hi; a++)
        for (int b = lo; b <= hi; b++) {
            int n = a * a + b * b;
            float want = n <= (1 << 24) ? sqrtf((float)n) : (float)sqrt((double)n);
            bad += hypotf((float)a, (float)b) != want;
        }
    return bad;
}
