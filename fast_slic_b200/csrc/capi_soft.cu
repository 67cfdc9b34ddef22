// fast_slic_b200/csrc/capi_soft.cu -- the extern "C" entry points of differentiable soft SLIC (soft_slic.cuh): the
// forward and backward of soft_assign, soft_pool and soft_unpool, and the hard labels of an association map.
// Stateless (device pointers; the caller provides every temporary), asynchronous on the caller's stream, never
// synchronise.
#include "capi_common.h"
#include "soft_slic.cuh"

#define SS_MAX_NODES (1LL << 30)

static bool ss_args_ok(int batch, int H, int W, int C, int nh, int nw) {
    return batch >= 0 && H >= 1 && W >= 1 && (long long)H * W <= MAX_IMAGE_PIXELS && C >= 1 && nh >= 1 && nh <= H &&
           nw >= 1 && nw <= W && (long long)nh * nw <= MAX_K && (long long)batch * nh * nw <= SS_MAX_NODES;
}

// Checks the arguments; returns 1 when there is work, 0 for an empty batch, or the (negative) error code
#define SS_BEGIN(batch, H, W, C, nh, nw, ...)                                                          \
    if (!ss_args_ok(batch, H, W, C, nh, nw)) return set_err(FSLIC_EINVAL, "bad batch, H, W, C or grid"); \
    if (batch == 0) return FSLIC_OK;                                                                  \
    {                                                                                                 \
        const void* req__[] = {__VA_ARGS__};                                                          \
        for (const void* r__ : req__)                                                                 \
            if (!r__) return set_err(FSLIC_EINVAL, "NULL argument");                                  \
    }                                                                                                 \
    USE_DEVICE(device);                                                                               \
    const SsGrid g = {H, W, C, nh, nw, nh * nw};                                                      \
    const long npx = (long)batch * H * W, ncell = (long)batch * g.K;                                  \
    cudaStream_t st = (cudaStream_t)stream;                                                           \
    (void)npx;                                                                                        \
    (void)ncell

// The block sums over every (image, cell, channel group): one warp each, 8 warps per CTA
template <int TERM>
static void ss_cell_sum(const SsGrid& g, long ncell, int device, cudaStream_t st, const float* w, const float* v,
                        const float* mu, float* out, float* z) {
    const long nwarps = ncell * ((g.C + SS_CG - 1) / SS_CG);
    k_ss_cell_sum<TERM><<<(int)grid_for(nwarps * 32, device), 256, 0, st>>>(g, nwarps, w, v, mu, out, z);
}

extern "C" int fslic_b200_soft_assign(int device, int batch, int H, int W, int C, int nh, int nw,
                                      const float* d_features, const float* d_centroids, float* d_assoc,
                                      void* stream) {
    SS_BEGIN(batch, H, W, C, nh, nw, d_features, d_centroids, d_assoc);
    k_ss_assign<<<(int)grid_for(npx, device), 256, 0, st>>>(g, npx, d_features, d_centroids, d_assoc);
    CK(cudaGetLastError());
    return FSLIC_OK;
}

extern "C" int fslic_b200_soft_assign_backward(int device, int batch, int H, int W, int C, int nh, int nw,
                                               const float* d_features, const float* d_centroids,
                                               const float* d_assoc, const float* d_grad_assoc, float* d_gd,
                                               float* d_grad_features, float* d_grad_centroids, void* stream) {
    SS_BEGIN(batch, H, W, C, nh, nw, d_features, d_centroids, d_assoc, d_grad_assoc, d_gd);
    k_ss_softmax_bwd<<<(int)grid_for(npx, device), 256, 0, st>>>(g, npx, d_assoc, d_grad_assoc, d_gd);
    if (d_grad_features)
        k_ss_unpool<SS_DIFF><<<(int)grid_for(npx, device), 256, 0, st>>>(g, npx, d_centroids, d_gd, d_features,
                                                                         d_grad_features);
    if (d_grad_centroids)
        ss_cell_sum<SS_DIFF>(g, ncell, device, st, d_gd, d_features, d_centroids, d_grad_centroids, nullptr);
    CK(cudaGetLastError());
    return FSLIC_OK;
}

extern "C" int fslic_b200_soft_pool(int device, int batch, int H, int W, int C, int nh, int nw, const float* d_values,
                                    const float* d_assoc, float* d_means, float* d_weights, void* stream) {
    SS_BEGIN(batch, H, W, C, nh, nw, d_values, d_assoc, d_means, d_weights);
    ss_cell_sum<SS_POOL>(g, ncell, device, st, d_assoc, d_values, nullptr, d_means, d_weights);
    CK(cudaGetLastError());
    return FSLIC_OK;
}

extern "C" int fslic_b200_soft_pool_backward(int device, int batch, int H, int W, int C, int nh, int nw,
                                             const float* d_values, const float* d_assoc, const float* d_means,
                                             const float* d_weights, const float* d_grad_means, float* d_grad_sums,
                                             float* d_grad_weights, float* d_grad_values, float* d_grad_assoc,
                                             void* stream) {
    SS_BEGIN(batch, H, W, C, nh, nw, d_values, d_assoc, d_means, d_weights, d_grad_means, d_grad_sums, d_grad_weights);
    k_ss_pool_grad<<<(int)grid_for(ncell, device), 256, 0, st>>>(g, ncell, d_grad_means, d_means, d_weights,
                                                                 d_grad_sums, d_grad_weights);
    if (d_grad_values)
        k_ss_unpool<SS_SUM><<<(int)grid_for(npx, device), 256, 0, st>>>(g, npx, d_grad_sums, d_assoc, nullptr,
                                                                        d_grad_values);
    if (d_grad_assoc)
        k_ss_slot_dot<<<(int)grid_for(npx, device), 256, 0, st>>>(g, npx, d_grad_sums, d_values, d_grad_weights,
                                                                  d_grad_assoc);
    CK(cudaGetLastError());
    return FSLIC_OK;
}

extern "C" int fslic_b200_soft_unpool(int device, int batch, int H, int W, int C, int nh, int nw, const float* d_values,
                                      const float* d_assoc, float* d_out, void* stream) {
    SS_BEGIN(batch, H, W, C, nh, nw, d_values, d_assoc, d_out);
    k_ss_unpool<SS_SUM><<<(int)grid_for(npx, device), 256, 0, st>>>(g, npx, d_values, d_assoc, nullptr, d_out);
    CK(cudaGetLastError());
    return FSLIC_OK;
}

extern "C" int fslic_b200_soft_unpool_backward(int device, int batch, int H, int W, int C, int nh, int nw,
                                               const float* d_values, const float* d_assoc, const float* d_grad_out,
                                               float* d_grad_values, float* d_grad_assoc, void* stream) {
    SS_BEGIN(batch, H, W, C, nh, nw, d_values, d_assoc, d_grad_out);
    if (d_grad_values) ss_cell_sum<SS_SUM>(g, ncell, device, st, d_assoc, d_grad_out, nullptr, d_grad_values, nullptr);
    if (d_grad_assoc)
        k_ss_slot_dot<<<(int)grid_for(npx, device), 256, 0, st>>>(g, npx, d_values, d_grad_out, nullptr, d_grad_assoc);
    CK(cudaGetLastError());
    return FSLIC_OK;
}

extern "C" int fslic_b200_soft_labels(int device, int batch, int H, int W, int nh, int nw, const float* d_assoc,
                                      uint16_t* d_labels, void* stream) {
    SS_BEGIN(batch, H, W, 1, nh, nw, d_assoc, d_labels);
    k_ss_argmax<<<(int)grid_for(npx, device), 256, 0, st>>>(g, npx, d_assoc, d_labels);
    CK(cudaGetLastError());
    return FSLIC_OK;
}
