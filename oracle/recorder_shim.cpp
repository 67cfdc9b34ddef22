// oracle/recorder_shim.cpp -- TEST INFRASTRUCTURE ONLY (never linked into the product).
//
// A thin extern "C" door into the UNMODIFIED reference sources (compiled in place by oracle/recorder.mk, output
// oracle/_ref/libfslic_ref_recorder.so) that drives every context the way cfast_slic.pyx:150-257 does with
// debug_mode = true and returns get_recorder_report() (context.h:75; recorder.h) -- the bytes SlicModel's
// last_recorder_report holds after the call.
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <string>
#include "context.h"
#include "lsc.h"
#include "arch/x64/avx2.h"

namespace {
template <typename Ctx>
std::string run(Ctx& ctx, uint16_t* out, int max_iter, float compactness, float min_size_factor, int stride,
                int convert_to_lab, int manhattan, int preemptive, float preemptive_thres, int num_threads) {
    ctx.num_threads = num_threads;
    ctx.compactness = compactness;
    ctx.min_size_factor = min_size_factor;
    ctx.subsample_stride_config = (int16_t)stride;
    ctx.convert_to_lab = convert_to_lab != 0;
    ctx.preemptive = preemptive != 0;
    ctx.preemptive_thres = preemptive_thres;
    ctx.manhattan_spatial_dist = manhattan != 0;
    ctx.debug_mode = true;
    ctx.initialize_state();
    ctx.iterate(out, max_iter);
    return ctx.get_recorder_report();
}
}  // namespace

extern "C" {

// kind: 0 = fslic::Context ("standard"), 1 = Context_X64_AVX2 ("x64/avx2"), 2 / 3 / 4 = ContextRealDist / ContextRealDistL2
// / ContextRealDistNoQ, 5 = ContextLSC ("standard").  clusters are read and updated in place, out gets the labels.
// Returns the report in a malloc'd buffer (free it with refr_free) and its length in *len.
char* refr_iterate(int kind, int H, int W, int K, const uint8_t* image, Cluster* clusters, uint16_t* out, int max_iter,
                   float compactness, float min_size_factor, int stride, int convert_to_lab, int manhattan, int preemptive,
                   float preemptive_thres, int num_threads, size_t* len) {
    std::string rep;
#define RUN(T)                                                                                                     \
    {                                                                                                              \
        T ctx(H, W, K, image, clusters);                                                                           \
        rep = run(ctx, out, max_iter, compactness, min_size_factor, stride, convert_to_lab, manhattan, preemptive, \
                  preemptive_thres, num_threads);                                                                  \
    }
    switch (kind) {
        case 0: RUN(fslic::Context) break;
        case 1: RUN(fslic::Context_X64_AVX2) break;
        case 2: RUN(fslic::ContextRealDist) break;
        case 3: RUN(fslic::ContextRealDistL2) break;
        case 4: RUN(fslic::ContextRealDistNoQ) break;
        default: RUN(fslic::ContextLSC) break;
    }
#undef RUN
    char* buf = static_cast<char*>(malloc(rep.size() + 1));
    memcpy(buf, rep.data(), rep.size() + 1);
    *len = rep.size();
    return buf;
}

void refr_free(char* p) { free(p); }

}  // extern "C"
