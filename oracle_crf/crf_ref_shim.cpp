// oracle_crf/crf_ref_shim.cpp -- TEST INFRASTRUCTURE ONLY: extern "C" doors into the UNMODIFIED reference SimpleCRF
// (src/simple-crf.{hpp,cpp}), driven through its C++ methods the way csimple_crf.pyx drives them.  The temporal energy
// goes through SimpleCRFFrame::calc_temporal_pairwise_energy with the other frame: the reference's C function
// simple_crf_frame_temporal_pairwise_energy passes the frame itself twice and always returns 0.
#include <stdint.h>
#include <cmath>  // simple-crf.hpp uses expf without including it (simple-crf.cpp includes <cmath> first)
#include <stdexcept>
#include <vector>
#include "simple-crf.hpp"

extern "C" {
int refc_sizeof_cluster() { return (int)sizeof(Cluster); }
void* refc_new(size_t C, size_t N) { return new SimpleCRF(C, N); }
void refc_free(void* c) { delete (SimpleCRF*)c; }
void refc_set_params(void* c, const SimpleCRFParams* p) { ((SimpleCRF*)c)->params = *p; }
int refc_push(void* c) { return ((SimpleCRF*)c)->push_frame().time; }
int refc_pop(void* c) { return ((SimpleCRF*)c)->pop_frame(); }
int refc_first(void* c) { return ((SimpleCRF*)c)->get_first_time(); }
int refc_last(void* c) { return ((SimpleCRF*)c)->get_last_time(); }
void refc_set_clusters(void* c, int t, const Cluster* cl) { ((SimpleCRF*)c)->get_frame(t).set_clusters(cl); }
// CSR -> the reference's Connectivity (num_nodes rows)
void refc_set_connectivity(void* c, int t, int rows, const int32_t* off, const uint32_t* nbr) {
    std::vector<int> counts(rows);
    std::vector<uint32_t*> lists(rows);
    for (int i = 0; i < rows; i++) {
        counts[i] = off[i + 1] - off[i];
        lists[i] = const_cast<uint32_t*>(nbr + off[i]);
    }
    Connectivity conn;
    conn.num_nodes = rows;
    conn.num_neighbors = counts.data();
    conn.neighbors = lists.data();
    ((SimpleCRF*)c)->get_frame(t).set_connectivity(&conn);
}
void refc_set_unary(void* c, int t, const float* u) { ((SimpleCRF*)c)->get_frame(t).set_unary(u); }
void refc_get_unary(void* c, int t, float* u) { ((SimpleCRF*)c)->get_frame(t).get_unary(u); }
void refc_set_unbiased(void* c, int t) { ((SimpleCRF*)c)->get_frame(t).set_unbiased(); }
void refc_set_mask(void* c, int t, const int* cls, float conf) { ((SimpleCRF*)c)->get_frame(t).set_mask(cls, conf); }
void refc_set_proba(void* c, int t, const float* p) { ((SimpleCRF*)c)->get_frame(t).set_proba(p); }
void refc_get_inferred(void* c, int t, float* q) { ((SimpleCRF*)c)->get_frame(t).get_inferred(q); }
void refc_reset_inferred(void* c, int t) { ((SimpleCRF*)c)->get_frame(t).reset_inferred(); }
void refc_initialize(void* c) { ((SimpleCRF*)c)->initialize(); }
void refc_inference(void* c, long long it) { ((SimpleCRF*)c)->inference((size_t)it); }
float refc_spatial(void* c, int t, int i, int j) { return ((SimpleCRF*)c)->get_frame(t).calc_spatial_pairwise_energy(i, j); }
float refc_temporal(void* c, int t, int i, int other) {
    SimpleCRF* crf = (SimpleCRF*)c;
    return crf->get_frame(t).calc_temporal_pairwise_energy(i, crf->get_frame(other));
}
}
