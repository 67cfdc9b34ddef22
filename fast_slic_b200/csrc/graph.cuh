// fast_slic_b200/csrc/graph.cuh -- consumers of the final label map (SURVEY.md section 8(f) rows 1-2), over a batch of
// label maps, one call per batch and no host synchronisation (so a CUDA graph can capture them).  Every image's result
// is what fast_slic_get_connectivity / fast_slic_get_mask_density / fast_slic_cluster_density_to_mask
// (fast-slic/src/fast-slic.cpp:16-78, 141-168) give for that image alone; the single-image entry points are batches of
// one.  fast_slic_knn_connectivity (:80-130) is not provided: it indexes its cell vector with a float expression that
// runs past the end for any centre low in the last cell row (:88), i.e. the reference itself has no defined result to
// match (oracle/slic_oracle.c).
#pragma once
#include "common.cuh"

#define CONN_EMPTY 0xffffffffu
#define CONNB_CHUNK 2048  // sorted pairs staged per round of k_connb_walk

// ---------------------------------------------------------------------------------------------
// Adjacency graph.  The reference scans the pixels in raster order; at every pixel it probes the right, lower and
// lower-right neighbour and links the two labels unless they are linked already or either list is full (12).  A
// refused link is refused again at every later probe (lists only grow), so the outcome is a function of the FIRST
// probe of every unordered label pair, taken in scan order:
//   k_connb_init      image b's table slice [b*T, (b+1)*T): keys empty, order (b << obits) | omax (omax = 2^obits - 1
//                     exceeds every probe order 3 * pixel + slot of an image), overflow flags cleared;
//   k_connb_discover  every probe whose labels differ files (b << obits) | (3 * pixel + slot) under its pair in its
//                     image's slice of an open-addressing hash table (CAS claims a slot, atomicMin keeps the first
//                     probe), so the image index never reorders pairs inside an image;
//   (radix sort)      one sort of all B*T slots over the obits + bbits bits in use: image b's slice stays at
//                     [b*T, (b+1)*T), its pairs in the order the reference first meets them, its empty slots after;
//   k_connb_walk      one CTA per image: the capacity rule with u8 counts in shared memory over the sorted pairs staged
//                     into shared memory a chunk at a time.  If the image's table overflowed (label maps with millions
//                     of distinct adjacent pairs) one thread replays the reference's loop itself over all pixels --
//                     slow, exact, never needed for superpixel maps -- chosen on the device from the image's flag.
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_connb_init(uint32_t* __restrict__ tkey, unsigned long long* __restrict__ tord,
                                                     long nslots, int tshift, int obits, int batch, int* __restrict__ overflow) {
    const unsigned long long omax = (1ull << obits) - 1ull;
    for (long s = (long)blockIdx.x * blockDim.x + threadIdx.x; s < nslots; s += (long)gridDim.x * blockDim.x) {
        tkey[s] = CONN_EMPTY;
        tord[s] = ((unsigned long long)(s >> tshift) << obits) | omax;
        if (s < batch) overflow[s] = 0;
    }
}

__global__ void __launch_bounds__(256) k_connb_discover(const uint16_t* __restrict__ labels, int batch, int H, int W, int K,
                                                         uint32_t* __restrict__ tkey, unsigned long long* __restrict__ tord,
                                                         uint32_t T, int obits, int* __restrict__ overflow) {
    const long per = (long)(H - 1) * (W - 1);
    const long n = per * batch;
    const uint32_t tmask = T - 1;
    for (long t = (long)blockIdx.x * blockDim.x + threadIdx.x; t < n; t += (long)gridDim.x * blockDim.x) {
        const long b = t / per, r = t - b * per;
        const int i = (int)(r / (W - 1)), j = (int)(r - (long)i * (W - 1));
        const long p = (long)i * W + j;
        const uint16_t* lab = labels + b * H * W;
        const uint32_t s = lab[p];
        if (s >= (uint32_t)K) continue;
        const uint32_t nb[3] = {lab[p + 1], lab[p + W], lab[p + W + 1]};
        uint32_t* key_slice = tkey + b * T;
        unsigned long long* ord_slice = tord + b * T;
#pragma unroll
        for (int u = 0; u < 3; u++) {
            const uint32_t g = nb[u];
            if (g >= (uint32_t)K || g == s) continue;
            if (u == 2 && (g == nb[0] || g == nb[1])) continue;  // same pair, later order: cannot be the first probe
            if (u == 1 && g == nb[0]) continue;
            const uint32_t key = s < g ? (s << 16 | g) : (g << 16 | s);
            const unsigned long long order = ((unsigned long long)b << obits) | ((unsigned long long)p * 3ull + (unsigned long long)u);
            uint32_t h = conn_hash(key) & tmask;
            int probes = 0;
            for (;;) {
                const uint32_t old = atomicCAS(&key_slice[h], CONN_EMPTY, key);
                if (old == CONN_EMPTY || old == key) {
                    atomicMin(&ord_slice[h], order);
                    break;
                }
                h = (h + 1) & tmask;
                if (++probes > 512) {
                    overflow[b] = 1;
                    break;
                }
            }
        }
    }
}

// grid = batch, dynamic shared memory = align16(K) + CONNB_CHUNK * 4.  sorted_key: the batch's tables sorted as above.
// Writes counts[b*K + k], neighbors[(b*K + k)*12 + v] (zero past the count) and, if replayed != NULL, replayed[b].
__global__ void __launch_bounds__(256) k_connb_walk(const uint32_t* __restrict__ sorted_key, uint32_t T,
                                                     const uint16_t* __restrict__ labels, int H, int W, int K,
                                                     const int* __restrict__ overflow, int32_t* __restrict__ counts,
                                                     uint32_t* __restrict__ neighbors, int32_t* __restrict__ replayed) {
    extern __shared__ __align__(16) unsigned char connb_smem[];
    uint8_t* cnt = connb_smem;
    uint32_t* chunk = reinterpret_cast<uint32_t*>(connb_smem + ((K + 15) & ~15));
    __shared__ int done;
    const int b = blockIdx.x;
    uint32_t* nbr = neighbors + (long)b * K * CONN_MAX;
    for (int k = threadIdx.x; k < K; k += blockDim.x) cnt[k] = 0;
    if (threadIdx.x == 0) done = 0;
    const int flagged = overflow[b];
    __syncthreads();
    if (flagged) {
        // fast-slic.cpp:29-74 by one thread, with the counts in shared memory
        if (threadIdx.x == 0) {
            const uint16_t* lab = labels + (long)b * H * W;
            for (int i = 0; i < H - 1; i++) {
                for (int j = 0; j < W - 1; j++) {
                    const long p = (long)i * W + j;
                    const uint32_t s = lab[p];
                    if (s >= (uint32_t)K) continue;
                    int ns = cnt[s];
                    const long probe[3] = {p + 1, p + W, p + W + 1};
                    for (int u = 0; u < 3; u++) {
                        const uint32_t g = lab[probe[u]];
                        if (g >= (uint32_t)K || g == s) continue;
                        const int ng = cnt[g];
                        if (ns >= CONN_MAX || ng >= CONN_MAX) continue;
                        bool exists = false;
                        for (int v = 0; v < ns && !exists; v++) exists = nbr[s * CONN_MAX + v] == g;
                        for (int v = 0; v < ng && !exists; v++) exists = nbr[g * CONN_MAX + v] == s;
                        if (exists) continue;
                        nbr[g * CONN_MAX + ng] = s;
                        cnt[g] = (uint8_t)(ng + 1);
                        nbr[s * CONN_MAX + ns] = g;
                        ns++;
                    }
                    cnt[s] = (uint8_t)ns;
                }
            }
        }
    } else {
        const uint32_t* keys = sorted_key + (long)b * T;
        for (uint32_t base = 0; base < T; base += CONNB_CHUNK) {
            for (int e = threadIdx.x; e < CONNB_CHUNK; e += blockDim.x)
                chunk[e] = base + e < T ? keys[base + e] : CONN_EMPTY;
            __syncthreads();
            if (threadIdx.x == 0) {
                int e = 0;
                for (; e < CONNB_CHUNK; e++) {
                    const uint32_t key = chunk[e];
                    if (key == CONN_EMPTY) break;  // (no pair key is all ones: a < b <= 65535)
                    const uint32_t a = key >> 16, c = key & 0xffffu;
                    const int na = cnt[a], nc = cnt[c];
                    if (na >= CONN_MAX || nc >= CONN_MAX) continue;  // fast-slic.cpp:43
                    nbr[a * CONN_MAX + na] = c;
                    nbr[c * CONN_MAX + nc] = a;
                    cnt[a] = (uint8_t)(na + 1);
                    cnt[c] = (uint8_t)(nc + 1);
                }
                if (e < CONNB_CHUNK) done = 1;
            }
            __syncthreads();
            if (done) break;
        }
    }
    __syncthreads();
    for (int k = threadIdx.x; k < K; k += blockDim.x) counts[(long)b * K + k] = cnt[k];
    for (int e = threadIdx.x; e < K * CONN_MAX; e += blockDim.x)
        if (e % CONN_MAX >= cnt[e / CONN_MAX]) nbr[e] = 0u;
    if (replayed && threadIdx.x == 0) replayed[b] = flagged ? 1 : 0;
}

// ---------------------------------------------------------------------------------------------
// Mask density (fast-slic.cpp:141-155) and broadcast (:157-168) over B images of n = H*W pixels and B*K clusters:
// sum[k] = sum of mask over the pixels labelled k; density = min(255, sum / max(num_members, 1)) -- num_members being
// the Cluster field (the last subsampled update's count), as in the reference.  Lanes holding the same label add once
// (MATCH.ANY + REDUX); a warp can straddle two (or, for n < 32, more) images, so the key carries the image index beside
// the label.
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_mask_sum_batch(const uint16_t* __restrict__ lab, const uint8_t* __restrict__ mask,
                                                         long n, int batch, int K, int32_t* __restrict__ sum) {
    const long total = n * batch;
    const long step = (long)gridDim.x * blockDim.x;
    const long nround = (total + step - 1) / step * step;  // whole warps stay in the loop: the warp intrinsics need all lanes
    for (long t = (long)blockIdx.x * blockDim.x + threadIdx.x; t < nround; t += step) {
        unsigned long long key = ~0ull;
        uint32_t v = 0;
        long slot = 0;
        if (t < total) {
            const uint32_t l = lab[t];
            v = mask[t];
            if (l < (uint32_t)K) {
                const long b = t / n;
                key = (unsigned long long)b << 16 | l;
                slot = b * K + l;
            }
        }
        const unsigned peers = __match_any_sync(FSLIC_FULL, key);
        const uint32_t s = __reduce_add_sync(peers, v);
        if (key != ~0ull && (threadIdx.x & 31) == (unsigned)(__ffs(peers) - 1) && s) atomicAdd(&sum[slot], (int)s);
    }
}

__global__ void k_density_final_batch(const int32_t* __restrict__ sum, const fslic_cluster* __restrict__ clusters, long nk,
                                      uint8_t* __restrict__ dens) {
    for (long k = (long)blockIdx.x * blockDim.x + threadIdx.x; k < nk; k += (long)gridDim.x * blockDim.x) {
        const uint32_t den = clusters[k].num_members > 1u ? clusters[k].num_members : 1u;
        const uint32_t v = (uint32_t)sum[k] / den;
        dens[k] = (uint8_t)(v < 255u ? v : 255u);
    }
}

__global__ void __launch_bounds__(256) k_density_broadcast_batch(const uint16_t* __restrict__ lab,
                                                                  const uint8_t* __restrict__ dens, long n, int batch, int K,
                                                                  uint8_t* __restrict__ out) {
    const long total = n * batch;
    for (long t = (long)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (long)gridDim.x * blockDim.x) {
        const uint32_t l = lab[t];
        out[t] = l < (uint32_t)K ? dens[t / n * K + l] : (uint8_t)0;
    }
}
