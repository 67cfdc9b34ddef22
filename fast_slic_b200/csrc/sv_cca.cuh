// fast_slic_b200/csrc/sv_cca.cuh -- connectivity enforcement of label volumes [B,D,H,W] (DESIGN.md section 4.22).
// The 2-D enforcer's rules (cca.cuh) lifted to 6-connectivity, with its selection heap replaced by a total order:
//   components   the 6-connected sets of equal labels, numbered by leader (smallest raster index) order
//   kept         the components of area >= min_size; of more than K, the K first by (area desc, leader asc)
//   labels       kept components take 0, 1, .. in leader order; component 0 takes 0 if not kept; every other component
//                takes the final label of the component of its leader's predecessor voxel (leader - 1 if x > 0, else
//                leader - W if y > 0, else leader - H*W)
//
// Kernels, all over the batch (every index below is local to its volume, N = D*H*W):
//   k_svc_runs     par[v] = the start of v's run of equal labels inside its warp's 32 columns of a row
//   k_svc_union    lock-free unions (atomicMin on roots, so a root is its set's minimum index) across warp seams in x
//                  and to the voxels above (y) and behind (z)
//   k_svc_flatten  par[v] = root; cid[v] = 1 at roots -- an exclusive scan of cid then numbers the components
//   k_svc_comp     integer areas (one atomicAdd per run of a warp), and each component's predecessor component
//   k_svc_select   one CTA per volume: counts the candidates; if more than K, a radix select of the K-th key; then the
//                  new labels of the kept components by a block scan in component order
//   k_svc_absorb   the other components walk their predecessor chains to a labelled component
//   k_svc_output   out[v] = the final label of v's component
#pragma once
#include "common.cuh"

#define SVC_SELECT_THREADS 1024

// The root of x: parents always have smaller indices, and a root is its own parent
__device__ __forceinline__ int svc_find(const int* par, int x) {
    int q = par[x];
    while (q != x) {
        x = q;
        q = par[x];
    }
    return x;
}

// Unites the sets of a and b, hanging the larger root under the smaller with atomicMin until one hang succeeds
__device__ __forceinline__ void svc_union(int* par, int a, int b) {
    a = svc_find(par, a);
    b = svc_find(par, b);
    while (a != b) {
        if (a < b) {
            const int t = a;
            a = b;
            b = t;
        }
        const int old = atomicMin(&par[a], b);
        if (old == a) break;  // a was still a root: done
        a = svc_find(par, old);  // a got another parent meanwhile: carry on from there
        b = svc_find(par, b);
    }
}

// One warp per 32 columns of a row (rows of every volume of the batch, nseg segments per row): a ballot of the lanes
// whose left neighbour in the warp has another label gives the run starts; par[v] = the start of v's run.
__global__ void __launch_bounds__(256) k_svc_runs(const uint16_t* __restrict__ labels, long rows, int W, int nseg,
                                                  long hwd, int* __restrict__ par) {
    const int lane = threadIdx.x & 31;
    const long warps = rows * nseg;
    for (long w = ((long)blockIdx.x * blockDim.x + threadIdx.x) >> 5; w < warps;
         w += ((long)gridDim.x * blockDim.x) >> 5) {
        const long row = w / nseg;
        const int x0 = (int)(w - row * nseg) * 32, x = x0 + lane;
        const long p = row * W + x;
        const uint32_t l = x < W ? (uint32_t)labels[p] : 0x10000u + lane;  // no label equals a lane past the row
        const uint32_t left = __shfl_up_sync(FSLIC_FULL, l, 1);
        const unsigned starts = __ballot_sync(FSLIC_FULL, lane == 0 || l != left);
        const int start = 31 - __clz(starts & (0xffffffffu >> (31 - lane)));
        if (x < W) {
            const long b = p / hwd;
            par[p] = (int)(p - b * hwd - lane + start);
        }
    }
}

// One thread per voxel: unions across the warp seams in x, with the voxel above and with the voxel behind.  A voxel
// whose left neighbour has its label skips the union above (behind) when the left neighbour's voxel above (behind) has
// it too: the left neighbour's run already joins the two runs.
__global__ void __launch_bounds__(256) k_svc_union(const uint16_t* __restrict__ labels, long total, int D, int H, int W,
                                                   int* __restrict__ par) {
    const long hw = (long)H * W, n = hw * D;
    for (long p = (long)blockIdx.x * blockDim.x + threadIdx.x; p < total; p += (long)gridDim.x * blockDim.x) {
        const long b = p / n;
        const int v = (int)(p - b * n);
        const int x = v % W, y = (v / W) % H, z = (int)(v / hw);
        const uint16_t l = labels[p];
        int* pv = par + b * n;
        const bool left = x > 0 && labels[p - 1] == l;
        if (left && (x & 31) == 0) svc_union(pv, v, v - 1);
        if (y > 0 && labels[p - W] == l && !(left && labels[p - W - 1] == l)) svc_union(pv, v, v - W);
        if (z > 0 && labels[p - hw] == l && !(left && labels[p - hw - 1] == l)) svc_union(pv, v, v - (int)hw);
    }
}

// par[v] = the root of v, flag[p] = 1 at roots (0 elsewhere), for the exclusive scan that numbers the components
__global__ void __launch_bounds__(256) k_svc_flatten(long total, long n, int* __restrict__ par, int* __restrict__ flag) {
    for (long p = (long)blockIdx.x * blockDim.x + threadIdx.x; p < total; p += (long)gridDim.x * blockDim.x) {
        const long b = p / n;
        const int v = (int)(p - b * n);
        const int r = svc_find(par + b * n, v);
        par[p] = r;
        flag[p] = r == v;
    }
}

// One thread per voxel, warps over consecutive voxels: area[g] of every component g (batch-wide component numbers
// cid[b*N + root]) by one integer atomicAdd per run of equal g in a warp, and at roots pred[g] = the component of the
// leader's predecessor voxel, -1 for the first component of a volume.
__global__ void __launch_bounds__(256) k_svc_comp(long total, int D, int H, int W, const int* __restrict__ par,
                                                  const int* __restrict__ cid, int* __restrict__ area,
                                                  int* __restrict__ pred) {
    const long hw = (long)H * W, n = hw * D;
    const int lane = threadIdx.x & 31;
    const long stride = (long)gridDim.x * blockDim.x;
    for (long base = ((long)blockIdx.x * blockDim.x + threadIdx.x) & ~31L; base < total; base += stride) {
        const long p = base + lane;
        int g = -1 - lane;  // distinct from every other lane's for a lane past the end
        if (p < total) {
            const long b = p / n;
            const int v = (int)(p - b * n), r = par[p];
            g = cid[b * n + r];
            if (r == v) {
                const int x = v % W, y = (v / W) % H;
                const long q = x > 0 ? v - 1 : y > 0 ? v - W : v >= hw ? v - hw : -1;
                pred[g] = q < 0 ? -1 : cid[b * n + par[b * n + q]];
            }
        }
        const unsigned same = __match_any_sync(FSLIC_FULL, g);
        if (p < total && lane == __ffs(same) - 1) atomicAdd(&area[g], __popc(same));
    }
}

// The exclusive prefix of `flag` over the block in thread order and the block total (all threads must call it)
__device__ __forceinline__ int svc_block_scan(int flag, int* s_warp, int& total) {
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = blockDim.x >> 5;
    const unsigned bal = __ballot_sync(FSLIC_FULL, flag);
    if (lane == 0) s_warp[wid] = __popc(bal);
    __syncthreads();
    if (wid == 0) {
        const int c = lane < nw ? s_warp[lane] : 0;
        int x = c;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int y = __shfl_up_sync(FSLIC_FULL, x, o);
            if (lane >= o) x += y;
        }
        if (lane < nw) s_warp[lane] = x - c;
        if (lane == 31) s_warp[32] = x;
    }
    __syncthreads();
    const int r = s_warp[wid] + __popc(bal & ((1u << lane) - 1));
    total = s_warp[32];
    __syncthreads();
    return r;
}

// The selection key of a candidate: smaller keys first, by area descending, then component number (leader) ascending
__device__ __forceinline__ unsigned long long svc_key(int area, int local) {
    return (unsigned long long)(0x7fffffffu - (uint32_t)area) << 32 | (uint32_t)local;
}

// One CTA per volume over its components [cid[b*N], cid[(b+1)*N]): fin[g] = the new label of a kept component, 0 for
// the first component, -1 for the others.  When more than K components reach min_size, a radix select (8 bits at a
// time, integer shared-memory histograms) finds the K-th smallest key, and the kept set is the keys up to it.
__global__ void __launch_bounds__(SVC_SELECT_THREADS) k_svc_select(long n, int K, int min_size,
                                                                   const int* __restrict__ cid,
                                                                   const int* __restrict__ area, int* __restrict__ fin) {
    __shared__ int s_warp[33];
    __shared__ int s_hist[256];
    __shared__ unsigned long long s_prefix;
    __shared__ int s_want;
    const int b = blockIdx.x;
    const int g0 = cid[(long)b * n], g1 = cid[(long)(b + 1) * n];
    int mine = 0;
    for (int g = g0 + threadIdx.x; g < g1; g += blockDim.x) mine += area[g] >= min_size;
#pragma unroll
    for (int o = 16; o; o >>= 1) mine += __shfl_xor_sync(FSLIC_FULL, mine, o);
    if ((threadIdx.x & 31) == 0) s_warp[threadIdx.x >> 5] = mine;
    __syncthreads();
    int ncand = 0;
    for (int w = 0; w < (int)(blockDim.x >> 5); w++) ncand += s_warp[w];
    __syncthreads();
    unsigned long long kth = ~0ull;
    if (ncand > K) {
        if (threadIdx.x == 0) {
            s_prefix = 0;
            s_want = K;
        }
        for (int shift = 56; shift >= 0; shift -= 8) {
            const unsigned long long hi = shift == 56 ? 0ull : ~0ull << (shift + 8);
            for (int d = threadIdx.x; d < 256; d += blockDim.x) s_hist[d] = 0;
            __syncthreads();
            const unsigned long long prefix = s_prefix;
            for (int g = g0 + threadIdx.x; g < g1; g += blockDim.x) {
                const int a = area[g];
                if (a < min_size) continue;
                const unsigned long long key = svc_key(a, g - g0);
                if ((key & hi) == prefix) atomicAdd(&s_hist[(int)(key >> shift) & 255], 1);
            }
            __syncthreads();
            if (threadIdx.x == 0) {
                int want = s_want, d = 0;
                for (; d < 255 && s_hist[d] < want; d++) want -= s_hist[d];
                s_want = want;
                s_prefix = prefix | (unsigned long long)d << shift;
            }
            __syncthreads();
        }
        kth = s_prefix;
    }
    int next = 0;
    for (int base = g0; base < g1; base += blockDim.x) {
        const int g = base + threadIdx.x;
        bool kept = false;
        if (g < g1) {
            const int a = area[g];
            kept = a >= min_size && svc_key(a, g - g0) <= kth;
        }
        int total;
        const int r = svc_block_scan(kept, s_warp, total);
        if (g < g1) fin[g] = kept ? next + r : g == g0 ? 0 : -1;
        next += total;
    }
}

// The components without a label, grid (blocks, volumes): each walks its predecessor chain (strictly decreasing
// component numbers) to the first component with a label, then writes that label along the walked chain.  Every write
// stores the one value the rules give that component, so a walk that meets another's write only ends sooner.
__global__ void __launch_bounds__(256) k_svc_absorb(long n, const int* __restrict__ cid, const int* __restrict__ pred,
                                                    int* fin) {
    const int b = blockIdx.y;
    const int g0 = cid[(long)b * n], g1 = cid[(long)(b + 1) * n];
    volatile int* vf = fin;
    for (int g = g0 + blockIdx.x * blockDim.x + threadIdx.x; g < g1; g += gridDim.x * blockDim.x) {
        if (vf[g] >= 0) continue;
        int h = pred[g];
        int label = vf[h];
        while (label < 0) {
            h = pred[h];
            label = vf[h];
        }
        for (int u = g; u != h; u = pred[u]) {
            if (vf[u] >= 0) break;
            vf[u] = label;
        }
    }
}

// out[p] = the final label of p's component
__global__ void __launch_bounds__(256) k_svc_output(long total, long n, const int* __restrict__ par,
                                                    const int* __restrict__ cid, const int* __restrict__ fin,
                                                    int16_t* __restrict__ out) {
    for (long p = (long)blockIdx.x * blockDim.x + threadIdx.x; p < total; p += (long)gridDim.x * blockDim.x) {
        const long b = p / n;
        out[p] = (int16_t)fin[cid[b * n + par[p]]];
    }
}
