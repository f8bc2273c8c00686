/*
 * sonet_b200.h — C-ABI of libsonet_b200.so, the H100 (sm_90a) implementation of SO-Net's
 * per-batch forward hot path (SURVEY.md §8).
 *
 * Conventions (all entry points):
 *   - extern "C", plain device pointers + int dims + a trailing cudaStream_t (passed as void*
 *     so that this header needs no CUDA include). No allocation, no synchronisation, no host
 *     round-trip inside: every call is CUDA-graph capturable. The caller allocates outputs.
 *   - All tensors are contiguous, channel-first, fp32 unless stated: [B, C, P] with P fastest.
 *   - Return value: 0 = SONET_OK, negative = error; sonet_last_error_string() describes the
 *     last error raised on the calling thread.
 *   - Pointers marked "nullable" may be NULL to skip that output.
 *
 * Each function cites the reference interface (file:line under lijx10/SO-Net) it replaces.
 */
#ifndef SONET_B200_H_
#define SONET_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SONET_OK 0
#define SONET_ERR_BAD_ARG (-1)
#define SONET_ERR_CUDA (-2)
#define SONET_ERR_UNSUPPORTED (-3)

typedef void* sonet_stream_t; /* cudaStream_t */

/* ---- library ------------------------------------------------------------------------------ */
const char* sonet_last_error_string(void);
/* "sonet_b200 <version> sm_90a" */
const char* sonet_version(void);

/* ---- a-6/a-7: per-node indexed arg-max pool ---------------------------------------------------
 * Replaces index_max.forward_cuda / forward_cuda_shared_mem
 *   (models/index_max_ext/index_max.cpp:132-148, index_max_cuda.cu:10-100; called at
 *   models/networks.py:181-185).
 * data [B,C,N] f32, index [B,N] i32 with values in [0,K) (validated only in debug builds; an
 * out-of-range value is clamped, never a wild write), out_idx [B,C,K] i32:
 *   out_idx[b,c,k] = lowest n with index[b,n]==k maximising data[b,c,n], provided that maximum
 *   is > -1000.0f; otherwise 0 (empty node, or all values <= -1000: the reference's sentinel).
 * out_val (nullable) [B,C,K] f32 = data[b,c,out_idx[b,c,k]]  — i.e. the masked gather of
 *   models/networks.py:185 (first_pn_out_masked_max) fused into the pool.
 * K <= 256 on the CUDA path. */
int sonet_index_max_f32(const float* data, const int32_t* index, int B, int C, int N, int K,
                        int32_t* out_idx, float* out_val, sonet_stream_t stream);

/* Host (CPU) variants kept because the reference module exports them
 * (index_max.forward_cpu / forward_multi_thread_cpu, index_max.cpp:33-112). They are API
 * surface of the plugin, not a fallback: the CUDA entry points never route here. Host pointers. */
int sonet_index_max_cpu_f32(const float* data, const int32_t* index, int B, int C, int N, int K,
                            int32_t* out_idx, int thread_num);

/* ---- a-1/a-2/a-3: SOM node <-> point assignment -------------------------------------------------
 * Replaces BatchSOM.query_topk (util/som.py:237-269) plus the cluster statistics and centre
 * lookup of Encoder.forward (models/networks.py:127-143, 168-172).
 * x [B,3,N], node [B,3,M]  (M <= 256, 1 <= k <= 4, k <= M)
 * Distances are ((dx*dx + dy*dy) + dz*dz) in fp32 without FMA contraction (bit-equal to the
 * reference's ((x-node)**2).sum(1)); the k nearest nodes are emitted in ascending distance,
 * lowest node index first on exact ties (the reference's topk(sorted=False) order is
 * implementation-defined: parity is per-point set equality).
 * Outputs:
 *   min_idx_i32 [B,k*N]  slot-major: [slot0 for all n | slot1 ... ] (util/som.py:261-266)
 *   min_idx_i64 [B,k*N]  nullable, same content as int64 (the dtype query_topk returns)
 *   count       [B,M] i32  = mask_row_sum (models/networks.py:128)
 *   row_max     [B,M] i32  = mask_row_max (count > 0)
 *   cluster_mean[B,3,M] f32 = sum_{assigned copies} x / (count + 1e-5f)   (networks.py:140-142)
 * count and cluster_mean are nullable together (then no statistics pass runs; row_max, if given,
 * is still filled — by the assignment kernel itself — which is all BatchSOM.query_topk needs).
 * The per-node sums are accumulated in a fixed order: results are bit-reproducible run to run
 * and independent of how the batch is sharded across GPUs. */
int sonet_som_assign(const float* x, const float* node, int B, int N, int M, int k,
                     int32_t* min_idx_i32, int64_t* min_idx_i64, int32_t* count,
                     int32_t* row_max, float* cluster_mean, sonet_stream_t stream);

/* BatchSOM.query_topk in ONE launch (util/som.py:237-269): assignment + dense one-hot mask
 * [B,k*N,M] i32 (written by the assignment kernel itself, a coalesced row per store) + mask_row_max
 * [B,M] i32 + min_idx as int64 (nullable) and int32. HBM-bound: 4*M*k bytes written per point. */
int sonet_som_query_topk(const float* x, const float* node, int B, int N, int M, int k,
                         int32_t* mask, int32_t* row_max, int64_t* min_idx_i64,
                         int32_t* min_idx_i32, sonet_stream_t stream);

/* Dense one-hot mask of the assignment, util/som.py:255-265: mask[b, s*N+n, m] =
 * (min_idx[b,s*N+n]==m), int32 [B,k*N,M]. Pure streaming write (HBM-bound). */
int sonet_som_mask(const int32_t* min_idx_i32, int B, int kN, int M, int32_t* mask,
                   sonet_stream_t stream);

/* Centre lookup + decentre + concat, models/networks.py:168-172.
 * centers[b,:,j] = cluster_mean[b,:,min_idx[b,j]] ; x_dec = x_stack - centers ;
 * x_aug = cat(x_dec, sn_stack) where x_stack/sn_stack are x/sn repeated k times along points.
 * x, sn [B,3,N] (sn nullable -> x_aug has 3 channels), outputs: centers [B,3,kN] (nullable),
 * x_aug [B,3+3,kN] (channels 0-2 are x_decentered). */
int sonet_som_decenter(const float* x, const float* sn, const float* cluster_mean,
                       const int32_t* min_idx_i32, int B, int N, int M, int k,
                       float* centers, float* x_aug, sonet_stream_t stream);

/* ---- e: the path's collective ------------------------------------------------------------------------
 * The eval forward shards over the batch with no exchange inside the path (SURVEY.md §8e); the
 * one collective is an all-gather of the per-shard result rows (logits [B/G, classes], per-cloud
 * losses) over NCCL/NVLink. NCCL is resolved from the running process (dlopen libnccl.so.2), so
 * the library itself links only libcudart.
 *   sonet_comm_unique_id: rank 0 fills a 128-byte NCCL unique id; the host program distributes it.
 *   sonet_comm_init: ncclCommInitRank on the CURRENT device -> opaque communicator.
 *   sonet_allgather: recv[r*bytes .. (r+1)*bytes) = rank r's send buffer, asynchronous on `stream`,
 *     CUDA-graph capturable; in-place (send == recv + rank*bytes) allowed.
 *   sonet_comm_nccl_version: NCCL version code, 0 when NCCL cannot be loaded. */
int sonet_comm_nccl_version(void);
int sonet_comm_unique_id(void* id128);
int sonet_comm_init(const void* id128, int rank, int world, void** comm_out);
int sonet_allgather(void* comm, const void* send, void* recv, long long bytes_per_rank,
                    sonet_stream_t stream);
int sonet_comm_destroy(void* comm);

/* ---- f-1: the auto-encoder's up-convolution decoder -------------------------------------------
 * Replaces UpConv.forward (models/layers.py:214-240; DecoderConv, models/networks.py:394-431):
 * nearest x2 up-sampling + 3x3 convolution (pad 1) + eval BatchNorm + ReLU, computed as four
 * parity GEMMs over the LOW-resolution map with K = 4*Cin (the 3x3 taps that coincide after
 * up-sampling are pre-summed by the host into four [Cout, 4*Cin] matrices, tap-major K).
 *   sonet_upconv_im2col_f32: in [B,Cin,H,W] -> xcol [4][B][4*Cin][H*W]: group g = py*2+px, tap
 *     t = a*2+c reads in[b, ci, i + a-1+py, j + c-1+px] (0 outside the map).
 *   sonet_pointwise_tc_pack_groups: G weight matrices [G,Cout,Cin] -> G consecutive wgmma blobs
 *     (sonet_pointwise_tc_blob_bytes(Cout,Cin) each) with one common pre-scale (*inv_scale).
 *   sonet_pointwise_tc_grouped_forward: out_g = act(inv_scale * W_g x_g + shift) for G groups in
 *     ONE launch. x [G*B, C, P]; with scat_w = W > 0 (G must be 4, P = H*W, P_out = 4P) row
 *     p = i*W + j of group (py,px) is stored at (2i+py)*2W + 2j+px of out [B,Cout,P_out]: the
 *     parity interleave of the up-convolution; otherwise group g writes out + g*out_gstride.
 *     splits > 1 divides K (number of 64-channel chunks must be divisible) across CTAs: raw partial
 *     sums go to scratch [G][splits][B][Cout][P] and a second kernel adds them in a fixed order,
 *     then shift / ReLU / scatter — for small maps, where one CTA per 128x256 output tile would
 *     leave most SMs idle while it streams K*256 weights alone. */
int sonet_upconv_im2col_f32(const float* in, int B, int Cin, int H, int W, float* xcol,
                            sonet_stream_t stream);
/* The im2col-free form for maps with H*W % 64 == 0 and Cin % 64 == 0: in [B,Cin,H,W] ->
 * out [3][B][Cin][H*W], the input shifted horizontally by -1, 0, +1 (zeros at the row ends);
 * sonet_pointwise_tc_grouped_forward(conv_w = W) then fetches tap (a,c) of parity (py,px) by TMA
 * from block c-1+px+1 at point coordinate p + (a-1+py)*W (vertical shifts are coordinate offsets
 * whose out-of-range part the TMA unit zero-fills): 3x the input is written instead of 16x. */
int sonet_upconv_hshift_f32(const float* in, int B, int Cin, int H, int W, float* out,
                            sonet_stream_t stream);
int sonet_pointwise_tc_pack_groups(const float* W, int G, int Cout, int Cin, void* blob_host,
                                   float* inv_scale);
int sonet_pointwise_tc_grouped_forward(const float* x, int C, int B, int P, const void* blob,
                                       long long blob_gstride, float inv_scale, const float* shift,
                                       int Cout, int relu, int groups, int splits, int scat_w,
                                       int conv_w, int P_out, long long out_gstride, float* out,
                                       float* scratch, sonet_stream_t stream);

/* ---- f-2: train-mode kernels of the point-wise layers ---------------------------------------------
 * EquivariantLayer in train() mode = Conv1d(k=1) -> MyBatchNorm1d with BATCH statistics
 * (models/layers.py:22-70, 282-296) -> ReLU, and its backward; the backward of the per-node pool
 * (the gather of models/networks.py:185).
 *   sonet_bn_train_forward_f32: x [B,C,P] -> per-channel batch mean / biased variance / invstd
 *     (two-stage, fp64 partial sums in a fixed order: bit-reproducible) and
 *     y = act(gamma*(x-mean)*invstd + beta) in one elementwise pass. partial: scratch of
 *     sonet_bn_partial_slots(B,C) doubles. (The running-statistics update with the reference's
 *     momentum schedule stays on the host side: two [C] vector ops.)
 *   sonet_bn_train_backward_f32: dy, x (the BN input) -> dx, dgamma, dbeta; with relu the gate is
 *     recomputed from x (gamma*xhat+beta > 0), so the forward output need not be kept.
 *   sonet_index_max_backward_f32: grad_data [B,C,N] = 0; grad_data[b,c,idx[b,c,k]] += grad_out[b,c,k]
 *     (k ascending, one thread per (b,c): deterministic also when empty nodes all gather point 0).
 *   sonet_pointwise_tc_pack_device: fp32 W [Cout,Cin] on the DEVICE -> wgmma blob (optionally of
 *     W^T, for the dgrad GEMM) with the power-of-two pre-scale computed on the device;
 *     scale2[0]=scale, scale2[1]=1/scale; scratch_bits: one uint32 of scratch.
 *   sonet_pointwise_tc_forward_dev: the generic wgmma layer with that blob (1/scale read from
 *     device memory): the forward GEMM y = W x + b and the dgrad GEMM dx = W^T dy of a training step.
 *   sonet_wgrad_tc_f32: the wgrad GEMM dW[co][ci] = sum_{b,p} dy[b,co,p] x[b,ci,p] on the same kernel:
 *     dy is transposed to [K = B*P][Cout] and every channel pre-scaled by its own power of two
 *     (gradients are far below fp16's normal range, and one layer's channels span many decades:
 *     each row of dW keeps fp32-order relative precision), x is packed as the weight operand with
 *     k = (b,p), K is split over CTAs (splits) and reduced in a fixed order. Result dWT [Cin][Cout].
 *     Device scratch: dyT sonet_wgrad_kpad(B,P,splits)*Cout floats, blob
 *     sonet_wgrad_blob_bytes(Cin,Kpad) bytes, part splits*Cin*Cout floats, small
 *     sonet_wgrad_small_floats(Cout) floats. Needs Cout % 64 == 0.
 *   sonet_absmax_scale_f32: scale2 = (s, 1/s), s the power of two with max|s*t| in [256,512). */
int sonet_bn_partial_slots(int B, int C);
int sonet_bn_train_forward_f32(const float* x, const float* gamma, const float* beta, int B, int C,
                               int P, float eps, int relu, double* partial, float* y,
                               float* save_mean, float* save_var, float* save_invstd,
                               sonet_stream_t stream);
int sonet_bn_train_backward_f32(const float* dy, const float* x, const float* mean,
                                const float* invstd, const float* gamma, const float* beta, int B,
                                int C, int P, int relu, double* partial, float* dx, float* dgamma,
                                float* dbeta, sonet_stream_t stream);
int sonet_index_max_backward_f32(const float* grad_out, const int32_t* idx, int B, int C, int N, int K,
                                 float* grad_data, sonet_stream_t stream);
int sonet_pointwise_tc_pack_device(const float* W, int Cout, int Cin, int transpose, void* blob,
                                   float* scale2, unsigned* scratch_bits, sonet_stream_t stream);
int sonet_pointwise_tc_forward_dev(const float* x0, int C0, int B, int P, const void* blob,
                                   const float* inv_scale_dev, const float* act_scale_dev,
                                   const float* shift, int Cout, int relu, int splits, float* out,
                                   float* scratch, sonet_stream_t stream);
int sonet_absmax_scale_f32(const float* t, long long n, float* scale2, unsigned* scratch_bits,
                           sonet_stream_t stream);
long long sonet_wgrad_kpad(int B, int P, int splits);
long long sonet_wgrad_blob_bytes(int Cin, long long Kpad);
long long sonet_wgrad_small_floats(int Cout);
int sonet_wgrad_tc_f32(const float* dy, const float* x, int B, int Cout, int Cin, int P, int splits,
                       float* dyT, void* blob, float* part, float* small, float* dWT,
                       sonet_stream_t stream);

/* ---- f-4: batch-SOM training --------------------------------------------------------------------
 * Replaces BatchSOM.batch_update / BatchSOM.optimize (util/som.py:295-366): T iterations of
 * {nearest-node assignment, per-node mean, neighbourhood-weighted node update} per cloud, in ONE
 * launch (a persistent CTA per cloud keeps cloud, nodes and assignment in shared memory).
 * x [B,3,N]; node_init [3,M] shared by every cloud (node_init_batched = 0; BatchSOM.node_init,
 * som.py:209-212) or [B,3,M] (node_init_batched = 1; a single batch_update on the current nodes);
 * weights [T,M,M] f32: weights[t][m][j] = get_weighting_matrix(sigma_t)[m] at grid cell j
 * (som.py:232-235); lr [T] f32. node_out [B,3,M] (may alias a batched node_init).
 * last_idx (nullable) [B,N] i32 = the assignment computed in the last iteration.
 * Numerics: distances bit-equal to ((x-node)**2).sum(1), first minimal node on ties
 * (torch.min); sums accumulated in fp64 in a fixed order and rounded once (the reference's
 * cascade torch.sum is ~1 ulp accurate; plain fp32 accumulation diverges through assignment
 * flips); mean = sum / (count + 1e-5f); node += sum_m ((mean_m - node_j) * occupied_m) * W[m][j] * lr.
 * M <= 256; N up to ~17k points with the cloud resident in shared memory (larger N re-reads x
 * through L2; N <= ~220k). */
int sonet_som_train(const float* x, const float* node_init, int node_init_batched,
                    const float* weights, const float* lr, int T, int B, int N, int M,
                    float* node_out, int32_t* last_idx, sonet_stream_t stream);

/* ---- f-3: on-device training augmentation of a batch ----------------------------------------------
 * Replaces the per-item numpy pipeline of the loader (data/modelnet_shrec_loader.py:218-247 over
 * data/augmentation.py:52-144) for all clouds at once: pc, sn [B,3,N] and som [B,3,M] (each
 * nullable together with its output) go through
 *   v = v . rot1[b] ; v = v . rot2[b]     rot1/rot2 [B,3,3] f64 row-major, nullable (identity)
 *   v += clip(sigma * g, -clip, clip)     per array (sigma <= 0: no jitter)
 *   v *= scale[b]                         [B] f64, nullable
 *   v += shift[b]                         [B,3] f64, nullable; points and SOM nodes only
 * in float64 like the loader, rounded to float32 once. The standard-normal draws g are either
 * given (noise_* [B,P,3] f64, DEVICE pointers: the loader's own numpy stream -> reproduces it) or,
 * when the pointer is NULL, generated in the kernel by Philox4x32-10 + Box-Muller keyed by
 * (seed, cloud, array, point). All matrices/vectors are device pointers. */
int sonet_augment_f32(const float* pc, const float* sn, const float* som, int B, int N, int M,
                      const double* rot1, const double* rot2, const double* scale,
                      const double* shift, double sigma_pc, double clip_pc, double sigma_sn,
                      double clip_sn, double sigma_som, double clip_som, const double* noise_pc,
                      const double* noise_sn, const double* noise_som, unsigned long long seed,
                      float* pc_out, float* sn_out, float* som_out, sonet_stream_t stream);

/* ---- a-4/a-5/a-8/a-9/a-10: point-wise shared MLP layer (1x1 conv + folded BN + ReLU) ---------
 * Replaces EquivariantLayer.forward / MyConv2d(1x1).forward in eval mode
 * (models/layers.py:203-210, 282-296): out[b,co,p] = act(scale[co]*sum_ci W[co,ci]*X[b,ci,p] +
 * shift[co] (+ addend[b,co,gidx[b,p]])), where X is the channel-concatenation of x0 [B,C0,P]
 * and x1 [B,C1,P] (x1 nullable with C1=0) — the concat of PointResNet (layers.py:431) and of
 * final_pointnet's input (networks.py:192) without materialising it.
 * Wt [C0+C1, Cout] row-major = the conv weight TRANSPOSED (so that a K-slab of weights is
 * contiguous along Cout), packed once by the host; scale/shift [Cout] hold conv bias and
 * eval-mode BatchNorm folded by the host (scale nullable = 1; the host may also fold scale into
 * Wt). relu: 0/1.
 * addend (nullable) [B,Cout,G] with gidx [B,P] i32 in [0,G): per-point gathered additive term,
 * used by the decomposed segmenter layer-1 (per-node and per-cloud channels, SURVEY §8a-10).
 * out [B,Cout,P]. (KNNModule's max over K, layers.py:365, is sonet_rowmax_f32 on the result.) */
int sonet_pointwise_layer_f32(const float* x0, int C0, const float* x1, int C1, int B, int P,
                              const float* Wt, const float* scale, const float* shift, int Cout,
                              int relu, const float* addend, const int32_t* gidx, int G,
                              float* out, sonet_stream_t stream);

/* MyLinear in eval mode (models/layers.py:155-166): out[b,co] = act(scale*(W[co,:].x[b,:]) + shift)
 * x [B,Cin], W [Cout,Cin], out [B,Cout]. */
int sonet_linear_f32(const float* x, int B, int Cin, const float* W, const float* scale,
                     const float* shift, int Cout, int relu, float* out, sonet_stream_t stream);

/* max over the last dim: in [R, L] -> out [R] (global max over nodes, networks.py:197). */
int sonet_rowmax_f32(const float* in, int R, int L, float* out, sonet_stream_t stream);

/* ---- a-8: kNN gather on SOM nodes -----------------------------------------------------------------
 * Replaces operations.knn_gather_wrapper / knn_gather_by_indexing (models/operations.py:19-54):
 * out[b,c,m,j] = src[b,c,idx[b,m,j]],  src [B,C,M], idx [B,M,Kstride] i64 (first K columns
 * used, as KNNModule slices precomputed_knn_I[:, :, 0:K], layers.py:332), out [B,C,M,K]. */
int sonet_knn_gather_f32(const float* src, const int64_t* idx, int B, int C, int M, int K,
                         int Kstride, float* out, sonet_stream_t stream);

/* KNNModule input assembly (models/layers.py:346-361) in one pass:
 * neighbours of node coordinates, their centre ('avg' = mean over K, 'center' = the node itself),
 * decentred neighbours, gathered neighbour features, concatenated:
 *   x_aug [B, 3+C, M*K], center [B,3,M].   center_type: 0 = 'avg', 1 = 'center'. */
int sonet_knn_assemble_f32(const float* coord, const float* feat, const int64_t* idx, int B, int C,
                           int M, int K, int Kstride, int center_type, float* center,
                           float* x_aug, sonet_stream_t stream);

/* Exact K-NN among the M nodes themselves (the precomputed_knn_I=None branch,
 * models/layers.py:334-337): ascending distance, lowest index on ties. idx [B,M,K] i64. */
int sonet_node_knn(const float* coord, int B, int M, int K, int64_t* idx, sonet_stream_t stream);

/* Per-point gather of node features (models/segmenter.py:90-98):
 * out[b,c,j] = src[b,c,gidx[b,j]], src [B,C,M], gidx [B,P] i32, out [B,C,P]. */
int sonet_gather_points_f32(const float* src, const int32_t* gidx, int B, int C, int M, int P,
                            float* out, sonet_stream_t stream);

/* mean over the k stacked copies (models/networks.py:331-336): in [B,C,k*N] -> out [B,C,N],
 * out = (1/k) * (in[...,0:N] + in[...,N:2N] (+ in[...,2N:3N])) in the reference's order. */
int sonet_kcopy_mean_f32(const float* in, int B, int C, int N, int k, float* out,
                         sonet_stream_t stream);

/* Segmentation loss of the segmenter wrapper (models/losses.py:30-43 CrossEntropyLossSeg.forward as
 * called by models/segmenter.py:129-131): mean (size_average=1) or sum over all points of
 * -log_softmax(score[b,:,n])[target[b,n]]; score [B,C,N] f32, target [B,N] int64. Targets equal to
 * -100 (NLLLoss's default ignore_index) do not count; any other out-of-range target yields NaN.
 * scratch: sonet_seg_loss_scratch_bytes(B, N) bytes of device memory; loss: one float (device). */
long long sonet_seg_loss_scratch_bytes(int B, int N);
int sonet_seg_loss_f32(const float* score, const long long* target, int B, int C, int N,
                       int size_average, void* scratch, float* loss, sonet_stream_t stream);

/* Part-segmentation IoU (models/losses.py:73-189 compute_iou_np_array / compute_iou, called by
 * part-seg/train.py:95). score [B,C,N] f32, seg [B,N] int64, label [B] int64; part table in CSR
 * form: category k owns part_ids[part_offsets[k] .. part_offsets[k+1]) (int32, table order), each
 * category 1..256 parts, every id in [0,C). pred = argmax over C (lowest class on ties, first NaN
 * wins); per part p of label[b]'s category, I = #(seg==p && pred==p), U = #(seg==p || pred==p),
 * iou = U ? I / (U + 0.0001) : 1.0 in double; iou_shape[b] [B] f64 = left-to-right sum / parts.
 * pred [B,N] int64 and correct [B] int32 (= #(pred == seg)) are nullable. Deterministic.
 * Device pointers; the table is not validated on the device: a label outside [0,num_categories)
 * yields iou_shape[b] = NaN. */
int sonet_seg_iou_f32(const float* score, const long long* seg, const long long* label, int B, int C,
                      int N, const int32_t* part_offsets, const int32_t* part_ids, int num_categories,
                      double* iou_shape, long long* pred, int32_t* correct, sonet_stream_t stream);
/* The same over host pointers, shapes split over at most thread_num threads (fewer for small
 * batches: at least 2^20 score elements per thread). Validates the table and every
 * label: a label outside the table returns SONET_ERR_BAD_ARG. */
int sonet_seg_iou_cpu_f32(const float* score, const long long* seg, const long long* label, int B,
                          int C, int N, const int32_t* part_offsets, const int32_t* part_ids,
                          int num_categories, double* iou_shape, long long* pred, int32_t* correct,
                          int thread_num);

/* SHREC'16 same-label retrieval ranking (shrec16/test.py:64-99). feature [Q,D] f32; label_in [Q]
 * int64, or NULL for the row argmax (lowest index on ties, first NaN wins). For each query q, the
 * items p with label p == label q (q included) ranked by d = float(sqrt(sum_j double(f_q[j] -
 * f_p[j])^2)) (fp32 differences, fp64 sum in index order), ascending, ties by ascending p, NaN last;
 * at most k of them. Outputs [Q,k]: idx int64 (p, -1 past count), dist f32 (NaN past count);
 * count [Q] int32 = min(group size, k), or -1 when the label is outside [0,L) (that item is nobody's
 * candidate); label_out [Q] int64 (nullable). Limits: 1 <= D <= 1024, 1 <= k <= 4096,
 * 1 <= L <= 4096, Q*k < 2^31. Deterministic. The device entry takes
 * sonet_retrieval_scratch_bytes(Q, D, L, k) bytes of 256-byte aligned device scratch, makes no
 * allocation and no host synchronisation; it returns -1 (bad arguments) from the size query. */
long long sonet_retrieval_scratch_bytes(int Q, int D, int L, int k);
int sonet_retrieval_rank_f32(const float* feature, const long long* label_in, int Q, int D, int L,
                             int k, void* scratch, long long scratch_bytes, long long* idx,
                             float* dist, int32_t* count, long long* label_out,
                             sonet_stream_t stream);
/* The same over host pointers, bit for bit, queries split over at most thread_num threads. */
int sonet_retrieval_rank_cpu_f32(const float* feature, const long long* label_in, int Q, int D, int L,
                                 int k, long long* idx, float* dist, int32_t* count,
                                 long long* label_out, int thread_num);
/* The bytes np.savetxt(f, rows, fmt='%06d %f') writes for each query's float64 rows
 * (ids[idx[q,i]], dist[q,i]), i < count[q]; host pointers, no file I/O. out == NULL: size query,
 * writes offsets [Q+1] (query q's text is out[offsets[q] .. offsets[q+1])) and returns the total.
 * Otherwise formats into out at those offsets (which must come from the size query) and returns
 * the total. Ids pass through double as numpy's float64 rows do; NaN prints "nan". Returns -1 when
 * a count is outside [0,k] or an idx outside [0,Q). */
long long sonet_retrieval_format_cpu(const long long* ids, const long long* idx, const float* dist,
                                     const int32_t* count, int Q, int k, long long* offsets,
                                     char* out, int thread_num);

/* ---- a-11: Chamfer distance ------------------------------------------------------------------------
 * Replaces ChamferLoss.forward (models/losses.py:237-290) including the Faiss IndexFlatL2
 * k=1 searches (losses.py:209-235) — exact brute force, direct differences, lowest index on ties.
 * pred [B,3,Mp], gt [B,3,N].
 *   idx_fwd [B,Mp] i32 : NN of each predicted point in gt;   idx_bwd [B,N] i32: NN of each gt
 *   point in pred  (either nullable)
 *   elem_fwd [B,Mp], elem_bwd [B,N] f32 (required): sqrt(|nn - p|^2 + 1e-8) per point
 *     (forward_loss_element / backward_loss_element, losses.py:281, 286)
 *   loss_fwd_arr, loss_bwd_arr [B] f32: per-cloud means of the above
 *   loss [3] f32: {forward_loss, backward_loss, forward_loss + backward_loss} (means over B).
 * All reductions run in a fixed order (bit-reproducible). */
int sonet_chamfer_f32(const float* pred, const float* gt, int B, int Mp, int N, int32_t* idx_fwd,
                      int32_t* idx_bwd, float* elem_fwd, float* elem_bwd, float* loss_fwd_arr,
                      float* loss_bwd_arr, float* loss, sonet_stream_t stream);

/* ---- a-5 on tensor cores: the whole first PointResNet as one wgmma kernel ----------------------
 * Replaces Encoder.first_pointnet = PointResNet(Cin,[64,128,256,384]).forward in eval mode
 * (models/layers.py:419-432, models/networks.py:82-83,176): three Conv1d(k=1)+BN+ReLU layers, the
 * skip-concat of layer-0's output and the bare 320->384 layer, for every stacked point copy.
 * Activations stay on chip between the layers: layer 0's output as a shared-memory operand image,
 * layers 1-2's outputs in registers as the next layer's wgmma A operand; fp32 parity comes from a
 * 3-product fp16 hi/lo split (see csrc/pointmlp_tc.cu).
 *   pack (host pointers): W0 [64,Cin], W1 [128,64], W2 [256,128], W3 [384,320] row-major with the
 *     eval BatchNorm scale already folded in; shift0..3 = folded bias/BN shift. Writes the fp16 hi/lo
 *     K-major core-matrix images streamed by the kernel into blob_host
 *     (sonet_pointresnet_tc_blob_bytes() bytes) and the fp32 side parameters into fparams_host
 *     (sonet_pointresnet_tc_fparam_count() floats).
 *   forward (device pointers): x [B,Cin,P] (Cin <= 6), blob/fparams as packed (blob 16-byte
 *     aligned), out [B,384,P].
 *   Range: the activations between the layers are split into fp16 hi/lo halves that each
 *   saturate at 65504, so an activation with |x| >= 131008 acts as +-131008 (the output stays
 *   finite); past 65504 precision drops to ~2^-12 of the term. Activations far below unit scale
 *   carry an absolute floor of 2^-25 each (error envelope: csrc/tc_common.cuh). */
int sonet_pointresnet_tc_blob_bytes(void);
int sonet_pointresnet_tc_fparam_count(void);
int sonet_pointresnet_tc_pack(const float* W0, int Cin, const float* W1, const float* W2,
                              const float* W3, const float* shift0, const float* shift1,
                              const float* shift2, const float* shift3, void* blob_host,
                              float* fparams_host);
int sonet_pointresnet_tc_forward(const float* x, int Cin, int B, int P, const void* blob,
                                 const float* fparams, float* out, sonet_stream_t stream);

/* Classifier-path fusion of the cluster statistics (models/networks.py:140-143), the node sort and
 * the decentring (networks.py:168-172) in ONE launch: a stable counting sort of the k*N stacked
 * copies by node, per-node coordinate sums in that fixed order (bit-reproducible, independent of
 * batch sharding), cluster_mean = sum / (count + 1e-5), then x_sorted / node_sorted / pos0 exactly
 * as sonet_som_sort_decenter defines them (rows of a node in ascending stacked order).
 * count [B,M] i32, cluster_mean [B,3,M] are outputs. Needs sonet_som_group_smem_bytes(N,M,k)
 * bytes of shared memory per block (4*k*N + small); fails with a message beyond the device limit.
 * When another 4*(6|3)*N bytes fit as well, the cloud (and its normals) is staged in shared memory.
 * sonet_som_group_mode: how sonet_som_group_decenter runs on a device with smem_optin bytes of
 * opt-in shared memory per block (cudaDevAttrMaxSharedMemoryPerBlockOptin): SONET_SOM_GROUP_STAGED,
 * SONET_SOM_GROUP_UNSTAGED, or SONET_SOM_GROUP_NONE (it would fail: M > 256, N >= 2^24 or too
 * little shared memory). with_sn: 1 when sn is passed. Negative on a bad argument. */
#define SONET_SOM_GROUP_NONE 0
#define SONET_SOM_GROUP_UNSTAGED 1
#define SONET_SOM_GROUP_STAGED 2
long long sonet_som_group_smem_bytes(int N, int M, int k);
int sonet_som_group_mode(int N, int M, int k, int with_sn, long long smem_optin);
int sonet_som_group_decenter(const float* x, const float* sn, const int32_t* min_idx_i32, int B,
                             int N, int M, int k, int32_t* count, float* cluster_mean,
                             float* x_sorted, int32_t* node_sorted, int32_t* pos0,
                             sonet_stream_t stream);
/* KNNModule input assembly (models/layers.py:346-361) directly from the fused pool's keys:
 * sonet_pool_finalize folded into sonet_knn_assemble_f32. Writes masked_max [B,C,M]
 * (first_pn_out_masked_max, models/networks.py:185), center [B,3,M], x_aug [B,3+C,M*K] and
 * resets the keys. M <= 256 and M*K <= 2304. */
int sonet_knn_assemble_pool_f32(const float* coord, int32_t* pool_keys, const float* p0,
                                const int64_t* idx, int B, int C, int M, int K, int Kstride,
                                int center_type, float* masked_max, float* center, float* x_aug,
                                sonet_stream_t stream);
/* ---- a-3 + a-5 + a-6/a-7 fused: node-sorted copies -> wgmma PointResNet -> per-node max -----
 * The classifier / auto-encoder path, where first_pn_out [B,384,kN] itself is never needed
 * (models/networks.py:168-185): it is neither written nor re-read.
 *   sonet_som_sort_decenter: buckets the k*N stacked copies of each cloud by node (order inside a
 *     node arbitrary) and writes, in that order, x_sorted [B,3(+3),kN] = decentred coordinates
 *     (+ normals), node_sorted [B,kN] i32 and pos0 [B] = sorted position of stacked copy 0.
 *     count [B,M] is sonet_som_assign's output.
 *   sonet_pointresnet_tc_pool_forward: as sonet_pointresnet_tc_forward on x_sorted, but instead of
 *     `out` it max-reduces every channel per node into pool_keys [B,384,M] i32 (order-preserving
 *     keys; must hold sonet_pool_keys_init()'s value on entry) and writes the 384 features of
 *     stacked copy 0 into p0 [B,384].
 *   sonet_pool_finalize: keys -> out_val [B,384,M] with the reference's semantics: the node's max
 *     if some copy exceeded the -1000 sentinel (index_max.cpp:80-81,103), else the feature of
 *     stacked copy 0 (the idx*mask_row_max gather of networks.py:185); resets the keys. */
int sonet_som_sort_decenter(const float* x, const float* sn, const float* cluster_mean,
                            const int32_t* min_idx_i32, const int32_t* count, int B, int N, int M,
                            int k, float* x_sorted, int32_t* node_sorted, int32_t* pos0,
                            sonet_stream_t stream);
int sonet_pointresnet_tc_pool_forward(const float* x_sorted, int Cin, int B, int P, const void* blob,
                                      const float* fparams, const int32_t* node_sorted,
                                      const int32_t* pos0, int M, int32_t* pool_keys, float* p0,
                                      sonet_stream_t stream);
int sonet_pool_keys_init(int32_t* keys, long long n, sonet_stream_t stream);
int sonet_pool_finalize(int32_t* keys, const float* p0, int B, int C, int M, float* out_val,
                        sonet_stream_t stream);

/* ---- a-8/a-9/a-10 on tensor cores: generic point-wise layer on wgmma --------------------------
 * Same contract as sonet_pointwise_layer_f32 (EquivariantLayer / MyConv2d 1x1 eval forward,
 * models/layers.py:203-210, 282-296) for layers dense enough for tensor cores (KNNModule,
 * final PointNet, segmenter head). fp32 parity through the fp16 hi/lo 3-product split.
 *   blob_bytes(Cout, Cin): size of the packed weight images.
 *   pack (host pointers): W [Cout,Cin] row-major fp32 with the BN scale folded in -> blob_host,
 *     *inv_scale = 1 / (power-of-two pre-scale applied to the weights).
 *   forward (device pointers): as sonet_pointwise_layer_f32 with (blob, inv_scale) instead of
 *     (Wt, scale).
 *   Range: each activation is split into fp16 hi/lo halves that each saturate at 65504, so an
 *   input with |x| >= 131008 acts as +-131008 (the output stays finite); past 65504 precision
 *   drops to ~2^-12 of the term. Error envelope (csrc/tc_common.cuh), per output:
 *   4e-6 * sum_k |W x| + 2^-24 * (sum_k |W| + sum_k |x| * inv_scale). */
long long sonet_pointwise_tc_blob_bytes(int Cout, int Cin);
int sonet_pointwise_tc_pack(const float* W, int Cout, int Cin, void* blob_host, float* inv_scale);
int sonet_pointwise_tc_forward(const float* x0, int C0, const float* x1, int C1, int B, int P,
                               const void* blob, float inv_scale, const float* shift, int Cout,
                               int relu, const float* addend, const int32_t* gidx, int G,
                               float* out, sonet_stream_t stream);
/* sonet_pointwise_tc_forward storing the point-major transpose: out [B,P,Cout], out[b,p,co] = the
 * value sonet_pointwise_tc_forward writes at [b,co,p], bit for bit. Consumers that gather whole
 * rows (the KNN module's per-node Y) read them as contiguous vectors. */
int sonet_pointwise_tc_forward_rows(const float* x0, int C0, const float* x1, int C1, int B, int P,
                                    const void* blob, float inv_scale, const float* shift, int Cout,
                                    int relu, const float* addend, const int32_t* gidx, int G,
                                    float* out, sonet_stream_t stream);

/* ---- KNNModule (3+C -> 512 -> 512, BN + ReLU, max over K) on wgmma, csrc/knn_tc.cu -----------
 * Layer 1 is split by linearity: Y = W1f x [B,512,M] (the C feature columns, computed once per
 * node by sonet_pointwise_tc_forward without shift or ReLU) is gathered per neighbour row and added
 * to W1d dec (the 3 coordinate columns, fp32). One kernel then runs layer 2 on wgmma and the max
 * over the K neighbours; neither h1 nor h2 is written.
 *   blob_bytes / pack (host pointers): W2 [512,512] folded fp32 -> blob_host, *inv_scale.
 *   forward (device pointers): coord [B,3,M], center [B,3,M] (as sonet_knn_assemble*_f32 writes
 *     it), idx [B,M,Kstride] int64 (first K columns), Y with element (b, c, n) at
 *     Y[b*512*M + c*y_cstride + n*y_nstride]: channel-major [B,512,M] (y_cstride = M,
 *     y_nstride = 1) or node-major [B,M,512] (1, 512; 8-byte aligned, read as float2 pairs, the
 *     faster layout), w1 [512][4] = {W1d[c,0..2], shift1[c]} (16-byte aligned), shift2 [512]
 *     -> out [B,512,M] = knn_feature_1. Both Y layouts give bit-identical results.
 *     2 <= K <= 16, M <= 65535. Error envelope of layer 2 as sonet_pointwise_tc_forward. */
long long sonet_knn_mlp_tc_blob_bytes(void);
int sonet_knn_mlp_tc_pack(const float* W2, void* blob_host, float* inv_scale);
int sonet_knn_mlp_tc_forward(const float* coord, const float* center, const int64_t* idx, int B,
                             int M, int K, int Kstride, const float* Y, long long y_cstride,
                             long long y_nstride, const float* w1, const void* blob,
                             float inv_scale, const float* shift2, float* out,
                             sonet_stream_t stream);

/* ---- opt-in fp16 mode of the eval wgmma entries (SONET_TC=fp16, INTEGRATION.md) ----------------
 * Each takes the arguments and the blob of the entry without the suffix, and runs every wgmma
 * GEMM as ONE fp16 product per MAC instead of the hi/lo split's three:
 *   y = (sum_k rn16sat(x_k) * rn16(s * w_k)) / s, accumulated in fp32,
 * where s is the blob's power-of-two pre-scale, rn16sat(x) the round-to-nearest fp16 of x saturated
 * at +-65504 (the split's hi word) and rn16(s * w) the hi image already in the blob. Everything
 * outside the GEMMs is unchanged: layer 0 of the PointResNet and layer 1's coordinate part of the
 * KNN module stay fp32 on CUDA cores, and so do all epilogues (shift, ReLU, addends, maxima,
 * scatter). Per output the rounding of both operands costs up to ~2^-10 * sum_k |w_k x_k|
 * (2^-11 each); against the rounded operands the GEMM is exact up to fp32 accumulation. Same
 * properties as the split entries: no allocation, no host synchronisation, deterministic, CUDA
 * graph capturable. */
int sonet_pointresnet_tc_forward_f16(const float* x, int Cin, int B, int P, const void* blob,
                                     const float* fparams, float* out, sonet_stream_t stream);
int sonet_pointresnet_tc_pool_forward_f16(const float* x_sorted, int Cin, int B, int P,
                                          const void* blob, const float* fparams,
                                          const int32_t* node_sorted, const int32_t* pos0, int M,
                                          int32_t* pool_keys, float* p0, sonet_stream_t stream);
int sonet_pointwise_tc_forward_f16(const float* x0, int C0, const float* x1, int C1, int B, int P,
                                   const void* blob, float inv_scale, const float* shift, int Cout,
                                   int relu, const float* addend, const int32_t* gidx, int G,
                                   float* out, sonet_stream_t stream);
int sonet_pointwise_tc_forward_rows_f16(const float* x0, int C0, const float* x1, int C1, int B,
                                        int P, const void* blob, float inv_scale,
                                        const float* shift, int Cout, int relu,
                                        const float* addend, const int32_t* gidx, int G, float* out,
                                        sonet_stream_t stream);
int sonet_pointwise_tc_grouped_forward_f16(const float* x, int C, int B, int P, const void* blob,
                                           long long blob_gstride, float inv_scale,
                                           const float* shift, int Cout, int relu, int groups,
                                           int splits, int scat_w, int conv_w, int P_out,
                                           long long out_gstride, float* out, float* scratch,
                                           sonet_stream_t stream);
int sonet_knn_mlp_tc_forward_f16(const float* coord, const float* center, const int64_t* idx,
                                 int B, int M, int K, int Kstride, const float* Y,
                                 long long y_cstride, long long y_nstride, const float* w1,
                                 const void* blob, float inv_scale, const float* shift2, float* out,
                                 sonet_stream_t stream);

/* ---- diagnostics -------------------------------------------------------------------------------
 * One 128 x N x K bf16 GEMM on wgmma (fp32 accumulate in registers), D = bf16(A) * bf16(Bm)^T.
 * A [128,K], Bm [N,K], D [128,N] fp32 row-major device pointers. mode 0: A from shared memory
 * (SS), 1: A from registers (RS). layout 0/1 selects which of the two canonical no-swizzle
 * K-major core-matrix arrangements is used; swap_fields exchanges the LBO/SBO descriptor fields.
 * Exists so that tests can pin the descriptor encodings the fused point-MLP kernel relies on. */
/* Same as sonet_pointresnet_tc_forward, additionally writing clock64() stamps of CTA 0 into
 * timeline64[128] (device): [126] kernel start, [127] kernel end. */
int sonet_debug_pointresnet_tc_timeline(const float* x, int Cin, int B, int P, const void* blob,
                                        const float* fparams, float* out, long long* timeline64,
                                        sonet_stream_t stream);
/* sonet_pointwise_tc_forward (single source, ReLU, no shift) with clock64() stamps of CTA 0 in
 * timeline128[128] (device): [127] kernel start, [126] kernel end. */
int sonet_debug_pointwise_tc_timeline(const float* x0, int C0, int B, int P, const void* blob,
                                      float inv_scale, int Cout, float* out, long long* timeline128,
                                      sonet_stream_t stream);
/* Cycles for `iters` back-to-back M=64 x N x 16 fp16 wgmmas issued by one warpgroup, B from shared
 * memory (no-swizzle K-major, 8-row-group stride `sbo`). mode 0: A from shared memory too, N = 64,
 * 96, 128 or 256; mode 1: A from registers, N = 96, 128 or 256. */
int sonet_debug_tc_mma_rate(int mode, int N, int sbo, int iters, long long* cycles,
                            sonet_stream_t stream);
/* sonet_pointresnet_tc_pool_forward with clock64() stamps of CTA 0 in timeline64[128] (device):
 * [126] kernel start, [127] kernel end, and per consumer warpgroup w and tile t < 6 of the CTA
 * [64 w + 10 t + phase]: phase 0 tile start, 1 act0 written, 2 layer 1 retired, 3 layer-2 epilogue
 * done, 4 + 2c layer-3 chunk c's last wgmma retired, 5 + 2c its pool epilogue done (c = 0..2).
 * [64 w + 60]: cycles warp 4w spent blocked on weight stages over all its tiles. Other slots are
 * not written. */
int sonet_debug_pointresnet_tc_pool_timeline(const float* x_sorted, int Cin, int B, int P,
                                             const void* blob, const float* fparams,
                                             const int32_t* node_sorted, const int32_t* pos0, int M,
                                             int32_t* pool_keys, float* p0, long long* timeline64,
                                             sonet_stream_t stream);
/* sonet_knn_mlp_tc_forward with clock64() stamps of CTA 0 in timeline128[128] (device): [126]
 * kernel start, [127] kernel end, and per consumer warpgroup w and work item i < 15 of the CTA
 * [64 w + 4 i + phase]: phase 0 item start, 1 first wgmma issued, 2 last wgmma retired, 3 neighbour
 * max and store done. */
int sonet_debug_knn_mlp_tc_timeline(const float* coord, const float* center, const int64_t* idx,
                                    int B, int M, int K, int Kstride, const float* Y,
                                    long long y_cstride, long long y_nstride, const float* w1,
                                    const void* blob, float inv_scale, const float* shift2,
                                    float* out, long long* timeline128, sonet_stream_t stream);
int sonet_debug_tc_probe(const float* A, const float* Bm, int N, int K, int mode, int layout,
                         int swap_fields, float* D, sonet_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* SONET_B200_H_ */
