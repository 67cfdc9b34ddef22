// oracle_euclid/euclid_ref_shim.cpp -- TEST INFRASTRUCTURE ONLY (never linked into the product).
//
// A thin extern "C" door into the UNMODIFIED reference sources (compiled in place by oracle_euclid/Makefile, outputs
// into oracle_euclid/_ref/) that drives them like cfast_slic.pyx does with `manhattan_spatial_dist = False`
// (cfast_slic.pyx:186,246; context.h:35): the default contexts of both archs, with and without `preemptive`, and the
// float-distance contexts.  The stage buffers are exposed like oracle/ref_shim.cpp does.
#include <cstdint>
#include "context.h"
#include "arch/x64/avx2.h"

namespace {
template <typename Base>
struct Probe : public Base {
    Probe(int H, int W, int K, const uint8_t* image, Cluster* clusters) : Base(H, W, K, image, clusters) {}
    void dump(uint8_t* quad_out, uint16_t* precca_out) {
        for (int i = 0; i < this->H; i++)
            for (int j = 0; j < this->W; j++) {
                if (quad_out)
                    for (int c = 0; c < 4; c++) quad_out[(i * this->W + j) * 4 + c] = this->quad_image.get(i, 4 * j + c);
                if (precca_out) precca_out[i * this->W + j] = this->assignment.get(i, j);
            }
    }
};

template <typename Ctx>
void run(Ctx& ctx, uint16_t* out, int max_iter, float compactness, float min_size_factor, int stride, int convert_to_lab,
         int preemptive, float preemptive_thres, int num_threads, uint8_t* quad_out, uint16_t* precca_out) {
    ctx.num_threads = num_threads;
    ctx.compactness = compactness;
    ctx.min_size_factor = min_size_factor;
    ctx.subsample_stride_config = (int16_t)stride;
    ctx.convert_to_lab = convert_to_lab != 0;
    ctx.preemptive = preemptive != 0;
    ctx.preemptive_thres = preemptive_thres;
    ctx.manhattan_spatial_dist = false;
    ctx.debug_mode = false;
    ctx.initialize_state();
    ctx.iterate(out, max_iter);
    ctx.dump(quad_out, precca_out);
}
}  // namespace

extern "C" {

int refe_sizeof_cluster() { return (int)sizeof(Cluster); }

// cfast_slic.pyx:124-147 (the seeding does not read the flag)
void refe_initialize(int H, int W, int K, const uint8_t* image, Cluster* clusters) {
    fslic::ContextBuilder builder("standard");
    fslic::Context* ctx = builder.build(H, W, K, image, clusters);
    ctx->initialize_clusters();
    delete ctx;
}

// cfast_slic.pyx:150-197 with manhattan_spatial_dist = False; arch: 0 = "standard", 1 = "x64/avx2".
// quad_out (u8[H*W*4]) and precca_out (u16[H*W]) may be NULL.
void refe_iterate(int arch, int H, int W, int K, const uint8_t* image, Cluster* clusters, uint16_t* out, int max_iter,
                  float compactness, float min_size_factor, int stride, int convert_to_lab, int preemptive,
                  float preemptive_thres, int num_threads, uint8_t* quad_out, uint16_t* precca_out) {
    if (arch == 1) {
        Probe<fslic::Context_X64_AVX2> ctx(H, W, K, image, clusters);
        run(ctx, out, max_iter, compactness, min_size_factor, stride, convert_to_lab, preemptive, preemptive_thres,
            num_threads, quad_out, precca_out);
    } else {
        Probe<fslic::Context> ctx(H, W, K, image, clusters);
        run(ctx, out, max_iter, compactness, min_size_factor, stride, convert_to_lab, preemptive, preemptive_thres,
            num_threads, quad_out, precca_out);
    }
}

// cfast_slic.pyx:198-252 with manhattan_spatial_dist = False: 0 = ContextRealDist, 1 = ContextRealDistL2, 2 = NoQ
void refe_iterate_real(int variant, int H, int W, int K, const uint8_t* image, Cluster* clusters, uint16_t* out,
                       int max_iter, float compactness, float min_size_factor, int stride, int convert_to_lab,
                       int num_threads, uint16_t* precca_out) {
    if (variant == 0) {
        Probe<fslic::ContextRealDist> ctx(H, W, K, image, clusters);
        run(ctx, out, max_iter, compactness, min_size_factor, stride, convert_to_lab, 0, 0.05f, num_threads, nullptr,
            precca_out);
    } else if (variant == 1) {
        Probe<fslic::ContextRealDistL2> ctx(H, W, K, image, clusters);
        run(ctx, out, max_iter, compactness, min_size_factor, stride, convert_to_lab, 0, 0.05f, num_threads, nullptr,
            precca_out);
    } else {
        Probe<fslic::ContextRealDistNoQ> ctx(H, W, K, image, clusters);
        run(ctx, out, max_iter, compactness, min_size_factor, stride, convert_to_lab, 0, 0.05f, num_threads, nullptr,
            precca_out);
    }
}

}  // extern "C"
