// oracle_lsc/lsc_ref_shim.cpp -- TEST INFRASTRUCTURE ONLY (never linked into the product).
//
// A thin extern "C" door into the UNMODIFIED reference sources (compiled in place by oracle_lsc/Makefile, outputs into
// oracle_lsc/_ref/) that drives ContextLSC like cfast_slic.pyx:198-252 does for real_dist_type 'lsc' with arch
// "standard" (lsc-builder.cpp), at any thread count.  A probe subclass exposes the protected feature buffers
// (lsc.h:9-14) through the one virtual hook map_image_into_feature_space and map_centroids_into_feature_space call,
// normalize_features (lsc.cpp:161,193,305):
//   * 1st call (image): the raw features and the weights are in place.  The reference keeps its ten feature means in a
//     local array (lsc.cpp:138-150); the probe recomputes them from the reference's own raw features with the
//     reference's expression -- one serial float sum per feature, divided by the pixel count -- so that the stage test
//     can pin them too.  The weights are the reference's.
//   * 2nd call (centroids): after it returns, centroid_features holds the initial centroid features.
//   * the centroid features at the end of iterate() are read after it returns.
#include <cstdint>
#include "lsc.h"

namespace {
struct Probe : public fslic::ContextLSC {
    Probe(int H, int W, int K, const uint8_t* image, Cluster* clusters) : fslic::ContextLSC(H, W, K, image, clusters) {}
    int calls = 0;
    float* means_out = nullptr;
    float* weights_out = nullptr;
    float* cinit_out = nullptr;

    void normalize_features(float* __restrict numers[10], float* __restrict weights, int size) override {
        if (calls == 0) {
            const int len = H * W;
            for (int f = 0; f < 10; f++) {
                float sum = 0;
                for (int i = 0; i < len; i++) sum += image_features[f][i];
                if (means_out) means_out[f] = sum / len;
            }
            if (weights_out)
                for (int i = 0; i < len; i++) weights_out[i] = image_weights[i];
        }
        fslic::ContextLSC::normalize_features(numers, weights, size);
        if (calls == 1 && cinit_out) dump_centroids(cinit_out);
        calls++;
    }
    void dump_centroids(float* out) {
        for (int k = 0; k < K; k++)
            for (int f = 0; f < 10; f++) out[k * 10 + f] = centroid_features[f][k];
    }
    void dump(uint16_t* precca_out) {
        if (precca_out)
            for (int i = 0; i < H; i++)
                for (int j = 0; j < W; j++) precca_out[i * W + j] = assignment.get(i, j);
    }
};
}  // namespace

extern "C" {

int refl_sizeof_cluster() { return (int)sizeof(Cluster); }

// cfast_slic.pyx:198-252 with real_dist_type 'lsc', arch "standard".  The stage outputs may be NULL: means float[10],
// weights float[H*W], cinit / cfinal float[K][10], precca u16[H*W].
void refl_iterate_lsc(int H, int W, int K, const uint8_t* image, Cluster* clusters, uint16_t* out, int max_iter,
                      float compactness, float min_size_factor, int stride, int convert_to_lab, int manhattan,
                      int num_threads, uint16_t* precca_out, float* means_out, float* weights_out, float* cinit_out,
                      float* cfinal_out) {
    Probe ctx(H, W, K, image, clusters);
    ctx.means_out = means_out;
    ctx.weights_out = weights_out;
    ctx.cinit_out = cinit_out;
    ctx.num_threads = num_threads;
    ctx.compactness = compactness;
    ctx.min_size_factor = min_size_factor;
    ctx.subsample_stride_config = (int16_t)stride;
    ctx.convert_to_lab = convert_to_lab != 0;
    ctx.preemptive = false;
    ctx.preemptive_thres = 0.05f;
    ctx.manhattan_spatial_dist = manhattan != 0;
    ctx.debug_mode = false;
    ctx.initialize_state();
    ctx.iterate(out, max_iter);
    ctx.dump(precca_out);
    if (cfinal_out) ctx.dump_centroids(cfinal_out);
}

}  // extern "C"
