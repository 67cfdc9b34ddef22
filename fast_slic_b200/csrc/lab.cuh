// fast_slic_b200/csrc/lab.cuh -- RGB -> CIELAB integer-LUT kernel and grid seeding.
#pragma once
#include "cellgrid.cuh"
#include "common.cuh"

struct LabConsts {
    int Cb[9];  // roundf(C * 65536), cielab.h:300-301
};

// Replaces FastCIELabCvt::convert + rgb_to_cielab (fast-slic/src/cielab.h:308-325,337-353)
// and the raw-RGB copy branch of iterate (context.cpp:118-127).
// One thread converts 4 consecutive pixels of the flattened [B*H*W] pixel stream: 12 input bytes
// (3 x LDG.32 when the base is 4-byte aligned) -> one 16-byte STG.128 of (L*2, a, b, 0) quads.
// Both tables live in shared memory as u16 (gamma <= 8192, lab_tbl <= 8192): 16.9 KB.
// HBM traffic: 3 B read + 4 B written per pixel.
__global__ void __launch_bounds__(256) k_rgb_to_quad(const uint8_t* __restrict__ rgb, uint32_t* __restrict__ quad,
                                                      long npix, const uint16_t* __restrict__ g_gamma,
                                                      const uint16_t* __restrict__ g_labtbl, LabConsts lc,
                                                      int convert_to_lab) {
    __shared__ uint16_t s_gamma[256];
    __shared__ uint16_t s_lab[8193 + 7];
    if (convert_to_lab) {
        for (int t = threadIdx.x; t < 256; t += blockDim.x) s_gamma[t] = g_gamma[t];
        for (int t = threadIdx.x; t < 8193; t += blockDim.x) s_lab[t] = g_labtbl[t];
        __syncthreads();
    }
    const bool aligned = ((reinterpret_cast<uintptr_t>(rgb) & 3) == 0);
    const long ngroups = (npix + 3) >> 2;
    for (long gidx = (long)blockIdx.x * blockDim.x + threadIdx.x; gidx < ngroups; gidx += (long)gridDim.x * blockDim.x) {
        const long p0 = gidx << 2;
        uint8_t c[12];
        if (aligned && p0 + 4 <= npix) {
            const uint32_t* src = reinterpret_cast<const uint32_t*>(rgb + 3 * p0);
            uint32_t w0 = ld_nc_u32(src), w1 = ld_nc_u32(src + 1), w2 = ld_nc_u32(src + 2);
#pragma unroll
            for (int t = 0; t < 4; t++) {
                c[t] = (w0 >> (8 * t)) & 0xff;
                c[4 + t] = (w1 >> (8 * t)) & 0xff;
                c[8 + t] = (w2 >> (8 * t)) & 0xff;
            }
        } else {
#pragma unroll
            for (int t = 0; t < 12; t++) c[t] = (3 * p0 + t < 3 * npix) ? rgb[3 * p0 + t] : 0;
        }
        uint32_t out[4];
#pragma unroll
        for (int t = 0; t < 4; t++) {
            const int R = c[3 * t], G = c[3 * t + 1], B = c[3 * t + 2];
            if (convert_to_lab) {
                const int sr = s_gamma[R], sg = s_gamma[G], sb = s_gamma[B];
                const int xr = (lc.Cb[0] * sr + lc.Cb[1] * sg + lc.Cb[2] * sb) >> 16;
                const int yr = (lc.Cb[3] * sr + lc.Cb[4] * sg + lc.Cb[5] * sb) >> 16;
                const int zr = (lc.Cb[6] * sr + lc.Cb[7] * sg + lc.Cb[8] * sb) >> 16;
                const int fx = s_lab[xr], fy = s_lab[yr], fz = s_lab[zr];
                const int ciel = 116 * fy - (16 << 13);
                const int ciea = 500 * (fx - fy) + (128 << 13);
                const int cieb = 200 * (fy - fz) + (128 << 13);
                // unsigned shift, unsigned subtract, then clamp as int -- exactly cielab.h:322-324
                const int l = min(max((int)((unsigned)ciel >> 12), 0), 255);
                const int a = min(max((int)(((unsigned)ciea >> 12) - 128u), 0), 255);
                const int b = min(max((int)(((unsigned)cieb >> 12) - 128u), 0), 255);
                out[t] = (uint32_t)l | ((uint32_t)a << 8) | ((uint32_t)b << 16);
            } else {
                out[t] = (uint32_t)R | ((uint32_t)G << 8) | ((uint32_t)B << 16);
            }
        }
        if (p0 + 4 <= npix && ((reinterpret_cast<uintptr_t>(quad + p0) & 15) == 0)) {
            *reinterpret_cast<uint4*>(quad + p0) = make_uint4(out[0], out[1], out[2], out[3]);
        } else {
#pragma unroll
            for (int t = 0; t < 4; t++)
                if (p0 + t < npix) quad[p0 + t] = out[t];
        }
    }
}

// Round-2 form of the Lab branch.  ncu on the kernel above (720p x 32): the LSU pipe sits at 86 % of its wavefront
// peak -- six u16 table gathers per pixel with 2.8-way bank conflicts on average -- and the ALU pipe at 65 %.
// Here the 256-entry gamma table is replicated 32 times in shared memory, word (v * 32 + lane): every lane reads its own
// bank, so the three gamma gathers of a pixel are conflict free (the 8193-entry Lab table cannot be replicated and
// keeps its conflicts); a thread converts 16 consecutive pixels per step: 3 x LDG.128 in, 4 x STG.128 out.
// Same integer arithmetic, same tables (cielab.h:308-325).  Needs 16-byte aligned bases; pixels beyond the last full
// group of 16 are converted one by one by the last thread.
#define LAB16_SMEM (256 * 32 * 4 + 8200 * 2)
__device__ __forceinline__ uint32_t lab_one_pixel(int sr, int sg, int sb, const uint16_t* s_lab, const LabConsts& lc) {
    const int xr = (lc.Cb[0] * sr + lc.Cb[1] * sg + lc.Cb[2] * sb) >> 16;
    const int yr = (lc.Cb[3] * sr + lc.Cb[4] * sg + lc.Cb[5] * sb) >> 16;
    const int zr = (lc.Cb[6] * sr + lc.Cb[7] * sg + lc.Cb[8] * sb) >> 16;
    const int fx = s_lab[xr], fy = s_lab[yr], fz = s_lab[zr];
    const int ciel = 116 * fy - (16 << 13);
    const int ciea = 500 * (fx - fy) + (128 << 13);
    const int cieb = 200 * (fy - fz) + (128 << 13);
    // unsigned shift, unsigned subtract, then clamp as int -- exactly cielab.h:322-324
    const int l = min(max((int)((unsigned)ciel >> 12), 0), 255);
    const int a = min(max((int)(((unsigned)ciea >> 12) - 128u), 0), 255);
    const int b = min(max((int)(((unsigned)cieb >> 12) - 128u), 0), 255);
    return (uint32_t)l | ((uint32_t)a << 8) | ((uint32_t)b << 16);
}

__global__ void __launch_bounds__(256) k_rgb_to_lab16(const uint8_t* __restrict__ rgb, uint32_t* __restrict__ quad, long npix,
                                                       const uint16_t* __restrict__ g_gamma,
                                                       const uint16_t* __restrict__ g_labtbl, LabConsts lc) {
    extern __shared__ __align__(16) unsigned char lab_smem[];
    uint32_t* s_gam = reinterpret_cast<uint32_t*>(lab_smem);                       // [256][32]
    uint16_t* s_lab = reinterpret_cast<uint16_t*>(lab_smem + 256 * 32 * 4);        // [8193]
    for (int t = threadIdx.x; t < 256 * 32; t += blockDim.x) s_gam[t] = g_gamma[t >> 5];
    for (int t = threadIdx.x; t < 8193; t += blockDim.x) s_lab[t] = g_labtbl[t];
    __syncthreads();
    const uint32_t* gam = s_gam + (threadIdx.x & 31);  // this lane's copy: gam[v * 32]
    const long ngroups = npix >> 4;
    const uint4* src = reinterpret_cast<const uint4*>(rgb);
    uint4* dst = reinterpret_cast<uint4*>(quad);
    for (long gi = (long)blockIdx.x * blockDim.x + threadIdx.x; gi < ngroups; gi += (long)gridDim.x * blockDim.x) {
        const uint4 w0 = __ldg(src + 3 * gi), w1 = __ldg(src + 3 * gi + 1), w2 = __ldg(src + 3 * gi + 2);
        const uint32_t w[12] = {w0.x, w0.y, w0.z, w0.w, w1.x, w1.y, w1.z, w1.w, w2.x, w2.y, w2.z, w2.w};
        uint32_t out[16];
#pragma unroll
        for (int t = 0; t < 16; t++) {
            // byte 3t + c of the 48-byte group
            const int o0 = 3 * t, o1 = 3 * t + 1, o2 = 3 * t + 2;
            const uint32_t R = (w[o0 >> 2] >> (8 * (o0 & 3))) & 0xffu;
            const uint32_t G = (w[o1 >> 2] >> (8 * (o1 & 3))) & 0xffu;
            const uint32_t B = (w[o2 >> 2] >> (8 * (o2 & 3))) & 0xffu;
            out[t] = lab_one_pixel((int)gam[R * 32], (int)gam[G * 32], (int)gam[B * 32], s_lab, lc);
        }
#pragma unroll
        for (int v = 0; v < 4; v++) dst[4 * gi + v] = make_uint4(out[4 * v], out[4 * v + 1], out[4 * v + 2], out[4 * v + 3]);
    }
    if (blockIdx.x == gridDim.x - 1 && threadIdx.x == blockDim.x - 1) {
        for (long p = ngroups << 4; p < npix; p++)
            quad[p] = lab_one_pixel((int)gam[rgb[3 * p] * 32], (int)gam[rgb[3 * p + 1] * 32], (int)gam[rgb[3 * p + 2] * 32], s_lab, lc);
    }
}

// Replaces BaseContext::initialize_clusters (fast-slic/src/context.cpp:43-97).
// One thread per (image, cluster): the grid centre, then the raw RGB sampled at the centre.  Runs once per model, not
// per iterate.
__global__ void k_init_clusters(const uint8_t* __restrict__ images, fslic_cluster* __restrict__ clusters, int H,
                                int W, int K, int B) {
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    const int b = blockIdx.y;
    if (k >= K || b >= B) return;
    int cy, cx;
    init_grid_centre(k, H, W, K, cy, cx);
    fslic_cluster c;
    c.y = (float)cy;
    c.x = (float)cx;
    // context.cpp:88 evaluates `W * clusters[k].y + clusters[k].x` on float operands -- one fused multiply-add under
    // the reference's build flags (setup.py:137-149, -mfma) -- and truncates: above 2^24 pixels that is not always
    // the exact pixel index.  Same arithmetic here (clamped into the image for memory safety only).
    const int base = min((int)__fmaf_rn((float)W, (float)cy, (float)cx), H * W - 1);
    const size_t img = ((size_t)b * H * W + (size_t)base) * 3;
    c.r = images[img];
    c.g = images[img + 1];
    c.b = images[img + 2];
    c.a = 0.f;
    c.number = (uint16_t)k;
    c.is_active = 1;
    c.is_updatable = 1;
    c.num_members = 0;
    clusters[(size_t)b * K + k] = c;
}
