/*
 * oracle_c.c — TEST INFRASTRUCTURE, NOT PRODUCT CODE.
 *
 * Plain-C CPU restatement of the integer/index parts of SO-Net's forward hot path, used only as
 * the checker in tests/, __graft_entry__.smoke() and bench.py's cpu_baseline leg. Nothing in
 * so-net_b200/ links or calls this file.
 *
 * Each function cites the reference (lijx10/SO-Net) lines it restates. Pinning: checked against
 * the reference's own compiled plugin (oracle/_ref, built from /root/reference in place) and the
 * reference Python run here, through tests/golden/ (see oracle/make_golden.py).
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

/* models/index_max_ext/index_max.cpp:73-112 (index_max_forward_cpu): triple loop b,c,n;
 * max_val initialised to -1000, max_idx to 0; strict '>' so the first maximum wins. */
void oracle_index_max(const float* data, const int32_t* index, int B, int C, int N, int K,
                      int32_t* max_idx) {
  float* max_val = (float*)malloc(sizeof(float) * (size_t)B * C * K);
  for (size_t i = 0; i < (size_t)B * C * K; ++i) {
    max_val[i] = -1000.0f;
    max_idx[i] = 0;
  }
  for (int b = 0; b < B; ++b)
    for (int c = 0; c < C; ++c)
      for (int n = 0; n < N; ++n) {
        const int k = index[(size_t)b * N + n];
        const float v = data[((size_t)b * C + c) * N + n];
        float* mv = &max_val[((size_t)b * C + c) * K + k];
        if (v > *mv) {
          *mv = v;
          max_idx[((size_t)b * C + c) * K + k] = n;
        }
      }
  free(max_val);
}

/* util/som.py:245-253 (BatchSOM.query_topk): diff = x - node; diff_norm = (diff**2).sum(dim=1);
 * topk(k, largest=False). The sum over the 3 channels is ((d0*d0 + d1*d1) + d2*d2) in fp32
 * (SURVEY.md §8c: bit-equal to the reference expression). Slot order here: ascending distance,
 * lowest node index on exact ties, +inf then NaN distances last (the reference's sorted=False
 * order is implementation defined -> parity is per-point set equality). Output slot-major like
 * util/som.py:261-266: min_idx[b, s*N + n]. Compile with -ffp-contract=off. */
void oracle_som_topk(const float* x, const float* node, int B, int N, int M, int k,
                     int32_t* min_idx, float* min_dist /* nullable, same layout */) {
  for (int b = 0; b < B; ++b) {
    const float* xb = x + (size_t)b * 3 * N;
    const float* nb = node + (size_t)b * 3 * M;
    for (int n = 0; n < N; ++n) {
      float bd[8];
      int bi[8];
      int filled = 0;
      for (int s = 0; s < k; ++s) {
        bd[s] = INFINITY;
        bi[s] = -1;
      }
      for (int m = 0; m < M; ++m) {
        const float d0 = xb[n] - nb[m], d1 = xb[N + n] - nb[M + m], d2 = xb[2 * N + n] - nb[2 * M + m];
        const float d = (d0 * d0 + d1 * d1) + d2 * d2;
        if (d < bd[k - 1]) {
          int s = k - 1;
          while (s > 0 && d < bd[s - 1]) {
            bd[s] = bd[s - 1];
            bi[s] = bi[s - 1];
            --s;
          }
          bd[s] = d;
          bi[s] = m;
          if (filled < k) ++filled;
        }
      }
      /* fewer than k finite distances: then the +inf nodes, then the NaN ones, by index (the
       * order of torch.topk / a stable sort with NaN last; a NaN point gets nodes 0..k-1) */
      for (int pass = 0; pass < 2; ++pass)
        for (int m = 0; m < M && filled < k; ++m) {
          const float d0 = xb[n] - nb[m], d1 = xb[N + n] - nb[M + m], d2 = xb[2 * N + n] - nb[2 * M + m];
          const float d = (d0 * d0 + d1 * d1) + d2 * d2;
          if (pass == 0 ? isinf(d) && d > 0 : isnan(d)) {
            bd[filled] = d;
            bi[filled++] = m;
          }
        }
      for (int s = 0; s < k; ++s) {
        min_idx[(size_t)b * k * N + (size_t)s * N + n] = bi[s];
        if (min_dist) min_dist[(size_t)b * k * N + (size_t)s * N + n] = bd[s];
      }
    }
  }
}

/* models/losses.py:209-235: faiss.IndexFlatL2 k=1 search == exact brute-force arg-min of the
 * squared L2 distance. Faiss is not vendored in the reference (README.md:31,40, no version
 * pin): restated as direct differences, lowest index on ties — "parity unpinned" at the Faiss
 * boundary for near-tie index choices (DESIGN.md); the loss value is insensitive to them.
 * query [3,Q], db [3,D] channel-first like the model tensors. */
void oracle_nn_search(const float* query, int Q, const float* db, int D, int32_t* idx,
                      float* dist2) {
  for (int q = 0; q < Q; ++q) {
    float best = INFINITY;
    int bi = 0;
    for (int d = 0; d < D; ++d) {
      const float d0 = query[q] - db[d], d1 = query[Q + q] - db[D + d],
                  d2 = query[2 * Q + q] - db[2 * D + d];
      const float v = (d0 * d0 + d1 * d1) + d2 * d2;
      if (v < best) {
        best = v;
        bi = d;
      }
    }
    idx[q] = bi;
    if (dist2) dist2[q] = best;
  }
}
