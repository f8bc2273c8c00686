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

/* Activation codes. Entries with an `int relu` argument read it as one of these (0 and 1 keep
 * their old meaning); any other value fails with SONET_ERR_BAD_ARG before a CUDA call.
 * ELU is nn.ELU(alpha=1): x > 0 ? x : expm1(x), computed in fp32 in every precision mode. */
#define SONET_ACT_NONE 0
#define SONET_ACT_RELU 1
#define SONET_ACT_ELU 2

/* ---- library ------------------------------------------------------------------------------ */
const char* sonet_last_error_string(void);
/* "sonet_b200 <version> sm_90a" */
const char* sonet_version(void);

/* ---- a-6/a-7: per-node indexed arg-max pool ---------------------------------------------------
 * Replaces index_max.forward_cuda / forward_cuda_shared_mem
 *   (models/index_max_ext/index_max.cpp:132-148, index_max_cuda.cu:10-100; called at
 *   models/networks.py:181-185).
 * data [B,C,N] f32, index [B,N] i32 with values in [0,K). The values are not validated: an id
 * outside [0,K) is read as min((unsigned)id, K-1), so a negative or too large id counts as node
 * K-1 and is never a wild write. A NaN in data is never an arg-max (strict '>').
 * out_idx [B,C,K] i32:
 *   out_idx[b,c,k] = lowest n with index[b,n]==k maximising data[b,c,n], provided that maximum
 *   is > -1000.0f; otherwise 0 (empty node, or all values <= -1000: the reference's sentinel).
 * out_val (nullable) [B,C,K] f32 = data[b,c,out_idx[b,c,k]]  — i.e. the masked gather of
 *   models/networks.py:185 (first_pn_out_masked_max) fused into the pool.
 * K <= 256 on the CUDA path. N == 0 writes zeros to both outputs (data and index may be null). */
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
 * nearest x2 up-sampling + 3x3 convolution (pad 1) + eval BatchNorm + ReLU / ELU, computed as four
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
/* Train-mode BatchNorm: the batch statistics of Bg clouds, of which the caller holds B (Bg = B in
 * one process; in data-parallel training the global batch, sharded over the ranks). Every sum goes
 * through one record per (cloud, channel), which depends on nothing but that cloud's values, so
 * the results are the same bits at every SM count, sharding and world size. (The running-statistics
 * update with the reference's momentum schedule stays on the host side: two [C] vector ops.)
 *   sonet_bn_cloud_partials_f32: one fp64 record per (b, c) of x [B,C,P], in a fixed order inside the
 *     cloud (P == 1: a thread per record; P <= 1024: a warp; longer: a 256-thread CTA).
 *       backward == 0: rec [B,C,SONET_BN_REC_FWD] = {pivot = x[b,c,0], sum d, sum d*d}, d = x - pivot;
 *         dy, mean, invstd, gamma, beta unused (may be null).
 *       backward != 0: rec [B,C,SONET_BN_REC_BWD] = {sum g, sum g*xhat}, xhat = (x-mean)*invstd,
 *         g = dy times the activation's derivative, recomputed from x at z = gamma*xhat+beta (ReLU:
 *         [z > 0]; ELU: z > 0 ? 1 : exp(z)), so the forward output need not be kept (dy, x, mean,
 *         invstd required; gamma, beta nullable).
 *   sonet_bn_sync_forward_f32: rec [Bg,C,3], the records of all Bg clouds in global order, folded in
 *     ascending cloud order onto cloud 0's pivot p (S1 = sum_b sum d_b + P (p_b - p),
 *     S2 = sum_b sum d_b^2 + 2 (p_b - p) sum d_b + P (p_b - p)^2) into the biased mean / var /
 *     invstd over n = Bg*P values, then y = act(gamma*(x-mean)*invstd + beta) of the local x [B,C,P].
 *   sonet_bn_sync_backward_f32: rec [Bg,C,2] in global order -> dbeta = sum g, dgamma = sum g*xhat
 *     (ascending clouds: the same on every rank) and dx of the local x with 1/n = 1/(Bg*P).
 * act: SONET_ACT_*. Fail with SONET_ERR_BAD_ARG before any CUDA call for a null pointer, B, C or Bg
 * outside [1, 65535], B > Bg, P < 1 or an unknown activation code. No allocation, no atomics, no
 * host synchronisation. */
#define SONET_BN_REC_FWD 3
#define SONET_BN_REC_BWD 2
int sonet_bn_cloud_partials_f32(const float* x, const float* dy, const float* mean,
                                const float* invstd, const float* gamma, const float* beta, int B,
                                int C, int P, int act, int backward, double* rec,
                                sonet_stream_t stream);
int sonet_bn_sync_forward_f32(const double* rec, const float* x, const float* gamma,
                              const float* beta, int Bg, int B, int C, int P, float eps, int act,
                              float* y, float* mean, float* var, float* invstd,
                              sonet_stream_t stream);
int sonet_bn_sync_backward_f32(const double* rec, const float* dy, const float* x, const float* mean,
                               const float* invstd, const float* gamma, const float* beta, int Bg,
                               int B, int C, int P, int act, float* dx, float* dgamma, float* dbeta,
                               sonet_stream_t stream);
int sonet_index_max_backward_f32(const float* grad_out, const int32_t* idx, int B, int C, int N, int K,
                                 float* grad_data, sonet_stream_t stream);
/* Train-mode BatchNorm of a ragged batch: x [C, ld] is a [1,C,L] layer output whose cloud b owns the
 * columns col_offsets[b] .. col_offsets[b+1] (device int64 [B+1], from 0 to L; k*offsets for the
 * first PointResNet's stacked copies). The statistics cover all L columns, so a cloud weighs its size.
 *   sonet_bn_cloud_partials_ragged_f32: record (b, c) of row c's columns of cloud b, into rec
 *     [B,C,SONET_BN_REC_FWD | _BWD]: the dense record of that row at P = its length, with the same
 *     pivot, walk and warp / CTA pattern (length 1: a thread; <= 1024: a warp; longer: a CTA).
 *   sonet_bn_ragged_forward_f32 / _backward_f32: the B records folded in ascending cloud order, record
 *     b standing for its own n_b = col_offsets[b+1] - col_offsets[b] values in the shift identity of
 *     sonet_bn_sync_forward_f32, over n = L values; then y = act(BN(x)) / dx, dgamma, dbeta over
 *     [1,C,L] (ld = L) with 1/n = 1/L. With B equal lengths P every output is the dense entries' bits.
 * The device clamps offsets into [0, ld] (common.cuh); callers refuse empty ranges and offsets that do
 * not run from 0 to L. Fail with SONET_ERR_BAD_ARG before any CUDA call for a null pointer, B or C
 * outside [1, 65535], L (ld) outside [1, 2^31) or an unknown activation code.
 *   sonet_index_max_ragged_backward_f32: the backward of sonet_index_max_ragged_f32's gather:
 *     grad [C, ld] = 0, then grad[c, col_offsets[b] + idx[b,c,m]] += grad_out[b,c,m], m ascending, one
 *     thread per (b, c) (index_max_backward's order), idx clamped into the cloud's columns. grad_out,
 *     idx [B,C,M]; M in [1, 256]. */
int sonet_bn_cloud_partials_ragged_f32(const float* x, const float* dy, const float* mean,
                                       const float* invstd, const float* gamma, const float* beta,
                                       int C, long long ld, const long long* col_offsets, int B,
                                       int act, int backward, double* rec, sonet_stream_t stream);
int sonet_bn_ragged_forward_f32(const double* rec, const long long* col_offsets, int B, const float* x,
                                const float* gamma, const float* beta, int C, long long L, float eps,
                                int act, float* y, float* mean, float* var, float* invstd,
                                sonet_stream_t stream);
int sonet_bn_ragged_backward_f32(const double* rec, const long long* col_offsets, int B,
                                 const float* dy, const float* x, const float* mean,
                                 const float* invstd, const float* gamma, const float* beta, int C,
                                 long long L, int act, float* dx, float* dgamma, float* dbeta,
                                 sonet_stream_t stream);
int sonet_index_max_ragged_backward_f32(const float* grad_out, const int32_t* idx,
                                        const long long* col_offsets, int B, int C, int M,
                                        long long ld, float* grad, sonet_stream_t stream);
/* Instance normalisation, nn.InstanceNorm1d/2d(C, affine=True) with track_running_stats=False
 * (models/layers.py:133, 179, 257): eval and train compute the same forward. For each
 * row r = b*C + c of z [B,C,P] (P = points, neighbour slots or pixels), the biased mean and
 * variance of the row, then y = act(gamma[c]*(z - mean)*invstd + beta[c]), invstd = 1/sqrt(var+eps).
 * Statistics are exact two-pass (mean, then sum (z-mean)^2) in fp64 in a fixed order:
 * bit-reproducible; a constant row gives y = act(beta) exactly. gamma, beta nullable (identity);
 * act: SONET_ACT_*. reduce folds a reduction of the activated rows into the same pass:
 *   SONET_REDUCE_NONE       out [B,C,P], may alias z; k unused
 *   SONET_REDUCE_KCOPY_MEAN out [B,C,P/k], the mean over k stacked copies, copy j of point n at
 *                           j*(P/k) + n, summed in the reference's order (models/networks.py:331-336):
 *                           0.5*(a+b), (1/3)*((a+b)+c)
 *   SONET_REDUCE_GROUP_MAX  out [B,C,P/k], the max over consecutive groups of k (the KNN module's
 *                           max over neighbours, models/layers.py:365)
 * save_mean, save_invstd (nullable together) [B,C]: the row statistics the BatchNorm backward
 * (sonet_bn_cloud_partials_f32 with backward = 1, then sonet_bn_sync_backward_f32, both with
 * B = Bg = 1) takes on the [1, B*C, P] view, which is the instance-norm backward of every row.
 * One read of z and one write of out for rows of P <= 16384 (staged on chip); longer rows read z
 * again. Fails with SONET_ERR_BAD_ARG before any CUDA call for P < 2 (PyTorch: "Expected more than
 * 1 spatial element"), an unknown act or reduce code, or P not divisible by k. */
#define SONET_REDUCE_NONE 0
#define SONET_REDUCE_KCOPY_MEAN 1
#define SONET_REDUCE_GROUP_MAX 2
int sonet_instance_norm_f32(const float* z, const float* gamma, const float* beta, int B, int C, int P,
                            float eps, int act, int reduce, int k, float* out, float* save_mean,
                            float* save_invstd, sonet_stream_t stream);
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

/* ---- f-2 (decoder): train-mode up-convolution -----------------------------------------------------
 * UpConv in train() mode (models/layers.py:214-240): nearest x2 up-sampling + 3x3 conv (pad 1) as the
 * four parity GEMMs of f-1, with weights folded and packed on the device every step, and its
 * backward. For input x [B,Cin,H,W], output z [B,Cout,2H,2W] and upstream gradient dz:
 *   forward  z = sonet_pointwise_tc_grouped_forward_dev(Wg, x) + b (conv bias, no activation)
 *   dgrad    dx[b,ci,i,j] = sum_{g,t,co} Wg[g][co][t*Cin+ci] dz[b,co,2(i-oy)+py,2(j-ox)+px],
 *            oy = a-1+py, ox = c-1+px: ONE GEMM with K = 16*Cout, the dgrad matrix times the
 *            operand D of sonet_upconv_dgrad_im2col_f32 (sonet_pointwise_tc_forward_dev)
 *   wgrad    dWg[g] = sum_{b,p} dz_g xcol_g^T per parity (sonet_wgrad_tc_f32; dz_g = dz[:,:,py::2,
 *            px::2], xcol_g = group g of sonet_upconv_im2col_f32), then dW by the adjoint fold.
 * Every entry validates its arguments (SONET_ERR_BAD_ARG before any CUDA call), allocates nothing,
 * does not synchronise and uses no atomics: two identical calls give identical bits.
 *   sonet_upconv_fold_weights_f32: adjoint = 0: W [Cout,Cin,3,3] -> out = Wg [4][Cout][4*Cin]
 *     (Wg[g][co][t*Cin+ci] = sum of the taps that (g, t) collects, rows then columns ascending)
 *     and/or out_dgrad = the dgrad matrix [Cin][16*Cout], element (ci, (g*4+t)*Cout+co) =
 *     Wg[g][co][t*Cin+ci] (either may be null, not both). adjoint = 1: in = dWT [4][4*Cin][Cout] (the
 *     per-parity wgrad results in sonet_wgrad_tc_f32's layout) -> out = dW [Cout,Cin,3,3], each tap
 *     the sum of its one entry per parity in ascending parity order; out_dgrad must be null.
 *   sonet_upconv_dgrad_im2col_f32: dz [B,Cout,2H,2W] -> D [B][16*Cout][H*W], row (g*4+t)*Cout+co,
 *     point i*W+j = dz[b,co,2(i-oy)+py,2(j-ox)+px] (0 outside the map). Row (g, t0 = (1-py)*2 +
 *     (1-px), co) is the parity plane dz_g.
 *   sonet_pointwise_tc_pack_groups_device: the device twin of sonet_pointwise_tc_pack_groups (same
 *     blobs and pre-scale): W [G][Cout][Cin] on the device -> G consecutive blobs, scale2 = (s, 1/s)
 *     of the one power-of-two pre-scale of all G matrices; scratch: SONET_ABSMAX_SLOTS floats.
 *   sonet_pointwise_tc_grouped_forward_dev: sonet_pointwise_tc_grouped_forward with its inverse
 *     pre-scale read from device memory (inv_scale_dev, e.g. scale2 + 1 of the pack above). */
#define SONET_ABSMAX_SLOTS 256
int sonet_upconv_fold_weights_f32(const float* in, int Cout, int Cin, int adjoint, float* out,
                                  float* out_dgrad, sonet_stream_t stream);
int sonet_upconv_dgrad_im2col_f32(const float* dz, int B, int Cout, int H, int W, float* d,
                                  sonet_stream_t stream);
int sonet_pointwise_tc_pack_groups_device(const float* W, int G, int Cout, int Cin, void* blob,
                                          float* scale2, float* scratch, sonet_stream_t stream);
int sonet_pointwise_tc_grouped_forward_dev(const float* x, int C, int B, int P, const void* blob,
                                           long long blob_gstride, const float* inv_scale_dev,
                                           const float* shift, int Cout, int relu, int groups,
                                           int splits, int scat_w, int conv_w, int P_out,
                                           long long out_gstride, float* out, float* scratch,
                                           sonet_stream_t stream);

/* ---- opt-in fp16 mode of the train wgmma entries (SONET_TRAIN_TC=fp16, INTEGRATION.md) ----------
 * One-product twins of the three train-mode GEMM entries: ConvTC's forward and dgrad
 * (sonet_pointwise_tc_forward_dev), UpConvTC's forward (sonet_pointwise_tc_grouped_forward_dev) and
 * every wgrad (sonet_wgrad_tc_f32). Each runs its GEMM as ONE fp16 product per MAC instead of the
 * hi/lo split's three:
 *   y = (sum_k rn16sat(s_x * x_k) * rn16(s_w * w_k)) / (s_x * s_w), accumulated in fp32,
 * where s_w is the power-of-two pre-scale of the weight operand (of the blob packed on the device;
 * the wgrad's own pack of x, whose operand is the saved activation) and s_x that of the activation
 * operand (act_scale_dev; the wgrad's per-channel dy scales), each capped at 2^126 as in the split
 * entries. rn16sat is the round-to-nearest fp16 saturated at +-65504, rn16 the hi image of the blob.
 * With s_x from sonet_absmax_scale_f32 no operand of any fp32 magnitude saturates; values below
 * ~2^-24 of their tensor's max become fp16 subnormals and lose relative precision. The caller's
 * inv_scale_dev = 1/(s_x * s_w) is one fp32 value: it underflows to 0 when max|w| * max|x| is below
 * about 2^-131 (every product then below fp32's normal range). Per output the
 * rounding costs up to ~2^-10 * sum_k |w_k x_k|; against the rounded operands the GEMM is exact up
 * to fp32 accumulation. NaN and +-inf follow the split entries' rules: the same saturation and
 * epilogue, and a NaN scale (an infinite gradient) makes its outputs NaN.
 *   sonet_pointwise_tc_forward_dev_f16: the arguments of sonet_pointwise_tc_forward_dev.
 *   sonet_pointwise_tc_grouped_forward_dev_f16: those of sonet_pointwise_tc_grouped_forward_dev and
 *     act_scale_dev, the activations' pre-scale (1 element of device memory, or null for none), whose
 *     inverse the caller folds into inv_scale_dev.
 *   sonet_wgrad_tc_f16: the arguments and scratch of sonet_wgrad_tc_f32 (sonet_wgrad_kpad,
 *     sonet_wgrad_blob_bytes and sonet_wgrad_small_floats size it); x's blob is written as hi images
 *     only, half the bytes, in the same layout, and dyT stays fp32 (the GEMM rounds it as it loads).
 * Same properties as the split entries: arguments validated before any CUDA call (SONET_ERR_BAD_ARG),
 * no allocation, no host synchronisation, deterministic, CUDA graph capturable. */
int sonet_pointwise_tc_forward_dev_f16(const float* x0, int C0, int B, int P, const void* blob,
                                       const float* inv_scale_dev, const float* act_scale_dev,
                                       const float* shift, int Cout, int relu, int splits,
                                       float* out, float* scratch, sonet_stream_t stream);
int sonet_pointwise_tc_grouped_forward_dev_f16(const float* x, int C, int B, int P, const void* blob,
                                               long long blob_gstride, const float* inv_scale_dev,
                                               const float* act_scale_dev, const float* shift,
                                               int Cout, int relu, int groups, int splits,
                                               int scat_w, int conv_w, int P_out,
                                               long long out_gstride, float* out, float* scratch,
                                               sonet_stream_t stream);
int sonet_wgrad_tc_f16(const float* dy, const float* x, int B, int Cout, int Cin, int P, int splits,
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
 * last_idx (nullable) [B,N] i32 = the assignment computed in the last iteration; with T = 0 the
 * assignment against node_init (the arithmetic of iteration 1), and node_out = node_init.
 * Numerics: distances bit-equal to ((x-node)**2).sum(1), first minimal node on ties
 * (torch.min); sums accumulated in fp64 in a fixed order and rounded once (the reference's
 * cascade torch.sum is ~1 ulp accurate; plain fp32 accumulation diverges through assignment
 * flips); mean = sum / (count + 1e-5f); node += sum_m ((mean_m - node_j) * occupied_m) * W[m][j] * lr,
 * that sum over m carried exactly (fp64 TwoSum) and rounded once to the nearest fp32.
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
/* sonet_augment_ragged_f32: sonet_augment_f32's per-point arithmetic over whole clouds: points [T, ld]
 * (ld >= 6) rows xyz | normal, cloud b the rows offsets[b] .. offsets[b+1] (device int64 [B+1],
 * clamped into [0, T]), and som [B,3,M] (nullable with som_out). rot1, rot2, scale, shift as there,
 * per cloud; the shift skips the normals. The jitter is always drawn in the kernel, keyed by (seed,
 * cloud, array, cloud-local row): cloud b's row n gets the draws of point n of cloud b in
 * sonet_augment_f32. Writes points_out [T, 6] and som_out. B in [1, 65535], T < 2^31. */
int sonet_augment_ragged_f32(const float* points, long long T, int ld, const long long* offsets, int B,
                             const float* som, int M, const double* rot1, const double* rot2,
                             const double* scale, const double* shift, double sigma_pc,
                             double clip_pc, double sigma_sn, double clip_sn, double sigma_som,
                             double clip_som, unsigned long long seed, float* points_out,
                             float* som_out, sonet_stream_t stream);

/* ---- f-3: the loader's random choice of points, from a dataset in device memory ----------------
 * Replaces the head of the loaders' __getitem__ for a whole batch: np.random.choice(P, N,
 * replace=False) (data/modelnet_shrec_loader.py:198,212; rule SUBSET) and the ShapeNet rule
 * (data/shapenet_loader.py:142-154; rule FILL: N < P as SUBSET, else the whole cloud in source
 * order followed by N-P uniform draws with replacement, so N == P is the cloud in order).
 * data [sum P, 6] f32 point-major (xyz | normal), offsets [S+1] i64 (cloud s is rows
 * offsets[s]..offsets[s+1]), labels [sum P] i32 (nullable, with seg_out), cloud_ids [B] i64: all
 * device pointers. Outputs pc_out, sn_out [B,3,N] and seg_out [B,N] i64 (the part labels).
 * indices [B,N] i32 (DEVICE, nullable): the source positions within each cloud, e.g. the loader's
 * own numpy draws (reproduces it bit for bit); values outside [0,P) are clamped to [0,P-1]. When
 * NULL, the kernel draws them from Philox4x32-10 keyed by (seed, batch position, point): SUBSET is
 * the distribution of permutation(P)[:N], the FILL draws are unbiased (Lemire). A cloud id outside
 * [0,S) is clamped; a cloud longer than max_P is read as its first max_P points; an empty cloud
 * gives zeros. SUBSET with P < N is outside the contract (the caller checks the counts): such a
 * cloud is filled as by FILL. Fails with SONET_ERR_BAD_ARG before any CUDA call for an unknown
 * rule, N < 1, B outside [0,65535], S < 1, max_P < 1, max_P > SONET_SAMPLE_MAX_P without indices,
 * labels/seg_out not both null or both given, or a null data/offsets/cloud_ids/pc_out/sn_out. */
#define SONET_SAMPLE_SUBSET 0
#define SONET_SAMPLE_FILL 1
#define SONET_SAMPLE_MAX_P 65536
int sonet_sample_points_f32(const float* data, const int64_t* offsets, int S, const int32_t* labels,
                            const int64_t* cloud_ids, int B, int N, int max_P, int rule,
                            const int32_t* indices, unsigned long long seed, float* pc_out,
                            float* sn_out, int64_t* seg_out, sonet_stream_t stream);

/* ---- area-weighted surface sampling of triangle meshes (data/sampler_matlab/sampler.m) ---------
 * B meshes as ragged device arrays: verts [total_V, 3] f64 with v_off [B+1] i64 (mesh b's vertices
 * are rows v_off[b]..v_off[b+1]), faces [total_F, 3] i32 with f_off [B+1] i64 (vertex indices local
 * to the mesh; outside [0, V) they are clamped to [0, V-1]), mesh_ids [B] i64. Output out [B*N, 6]
 * f32, point-major xyz | normal, mesh b owning rows b*N .. b*N+N-1; face_out [B*N] i32 (nullable):
 * the mesh-local face of each point; area_out [B] f64 (nullable): each mesh's total area.
 * Arithmetic is float64, explicitly rounded (no FMA), rounded to f32 once:
 *   e1 = b - a, e2 = c - a, n = cross(e1, e2), |n| = sqrt((nx*nx + ny*ny) + nz*nz),
 *   area = 0.5 * |n|, normal = n / |n|; weight = area, or 0 when the area is 0 or not finite.
 * CDF: every sum sequential from +0, blocked by SONET_MESH_RUN faces per run and SONET_MESH_TILE
 * faces per tile (both starting at face 0 of the mesh): run[f] = inclusive sum of the weights of
 * f's run up to f; roff = sum of the totals of the preceding runs of f's tile; toff = sum of the
 * totals of the preceding tiles; cdf[f] = toff + (roff + run[f]); total = cdf[F-1].
 * Per sample with draws (r, u, v) in [0,1): t = r * total, face = the first f with cdf[f] > t,
 * clamped to the last face of positive weight; if u + v > 1 then u = 1-u, v = 1-v; the point is
 * (a + u*e1) + v*e2, uniform on the triangle (sampler.m:35's a + u*b + v*c is not a point of the
 * triangle and is not reproduced). draws [B*N, 3] f64 (DEVICE, nullable) are given (r, u, v);
 * when NULL, Philox4x32-10 keyed by (seed, mesh_ids[b], sample) draws 53-bit uniforms, so a mesh's
 * points do not depend on the batch it is sampled in.
 * area_out[b] is the total, or NaN when a face's area is not finite (or the mesh exceeds 2^31-1
 * faces or vertices); a mesh whose total is 0 or not finite writes NaN rows (face_out -1) and does
 * not affect the other meshes. The entry takes sonet_mesh_sample_scratch_bytes(B, total_F) bytes
 * of 256-byte aligned device scratch (the f64 CDF and per-tile and per-mesh state), allocates
 * nothing, does not synchronise, and is deterministic. Fails with SONET_ERR_BAD_ARG before any
 * CUDA call for B < 0, N outside [1, SONET_MESH_MAX_N], total_F or total_V outside [0, 2^40], a null
 * v_off/f_off/mesh_ids/scratch/out, null verts (faces) with total_V (total_F) > 0, or too small or
 * misaligned a scratch; B = 0 then returns without a launch. The size query returns -1 for bad
 * arguments. */
#define SONET_MESH_RUN 8
#define SONET_MESH_TILE 2048
#define SONET_MESH_MAX_N 16777216
long long sonet_mesh_sample_scratch_bytes(int B, long long total_F);
int sonet_mesh_sample_f32(const double* verts, const int64_t* v_off, long long total_V,
                          const int32_t* faces, const int64_t* f_off, long long total_F,
                          const int64_t* mesh_ids, int B, int N, const double* draws,
                          unsigned long long seed, void* scratch, long long scratch_bytes, float* out,
                          int32_t* face_out, double* area_out, sonet_stream_t stream);

/* ---- point clouds without normals: exact k-NN within each cloud, and PCA surface normals ---------
 * Input: data [T, stride] f32 point-major (xyz in columns 0..2, stride >= 3; a DeviceDataset's
 * [T, 6] works in place), offsets [S+1] i64 (cloud s is rows offsets[s]..offsets[s+1]), all device
 * pointers. Every offset is clamped into [0, T] and a decreasing pair is an empty cloud, so no
 * offsets value reads or writes out of range; a cloud's results do not depend on the other clouds.
 *
 * sonet_point_knn_f32: idx [T, K] i32, the cloud-local indices of each point's K nearest points of
 * its own cloud (the point itself included), dist [T, K] f32 (nullable) their distances
 * d = ((dx*dx + dy*dy) + dz*dz), dx = q.x - p.x etc., fp32, explicitly rounded, no FMA (the SOM
 * assignment's and sonet_node_knn's convention). Ascending distance, lowest index first on ties;
 * a NaN distance ranks after every other, +inf included, again by index. Every index lies in
 * [0, P); when P < K, slots P..K-1 hold -1 and dist +inf. Brute force over each cloud's P^2 pairs.
 *
 * sonet_point_normals_f32: from idx [T, K] (sonet_point_knn_f32's), per point: the neighbours with
 * an index in [0, P) give a mean and a centred covariance (divided by their count) in fp64, two
 * passes in slot order, explicitly rounded; the eigenvector of the smallest eigenvalue (cyclic
 * Jacobi in fp64) normalised in fp64 and rounded to f32 once is the normal, written to
 * normals + row * normal_stride (normal_stride >= 3, e.g. data + 3 with stride 6 for data[:, 3:6]);
 * curvature [T] (nullable) = l0 / (l0 + l1 + l2), the surface variation. A neighbourhood with fewer
 * than 3 neighbours, a non-finite neighbour coordinate, a covariance trace that is 0 or not finite,
 * or collinear neighbours (l1 <= 2^-40 (l0 + l1 + l2)) gives the zero vector and NaN curvature.
 * Sign: canonically, the component of largest magnitude of the f32 normal is positive (the first
 * such component on ties); then, with ref per orientation code, the normal flips iff
 * dot(n, ref) < 0, computed in fp64 ((nx*rx + ny*ry) + nz*rz); a dot of 0 or NaN keeps the
 * canonical sign:
 *   SONET_NORMALS_CANONICAL           no ref;
 *   SONET_NORMALS_AWAY_FROM_CENTROID  ref = p - c, c the cloud's fp64 mean: with 256 lanes, lane t
 *                                     sums rows t, t+256, .. in order from +0, then s[i] += s[i+h]
 *                                     for h = 128, 64, .., 1, and c = s[0] / P;
 *   SONET_NORMALS_TOWARD_VIEWPOINT    ref = view[s] - p, view [S, 3] f32 (one point per cloud).
 * The centroid code takes sonet_point_normals_scratch_bytes(S) bytes of 256-byte aligned device
 * scratch (nullable with the other codes).
 *
 * Both entries allocate nothing, do not synchronise, are deterministic and capturable in a CUDA
 * graph. They fail with SONET_ERR_BAD_ARG before any CUDA call for S < 0, T < 0, stride < 3, K outside
 * [3, SONET_POINT_KNN_MAX_K], a null offsets/idx (knn) or offsets/normals (normals), null data
 * (and idx) with T > 0, an unknown orientation code, a null view with the viewpoint code,
 * normal_stride < 3, or a missing, too small or misaligned scratch with the centroid code; S = 0
 * then returns without a launch. The size query returns -1 for S < 0. */
#define SONET_POINT_KNN_MAX_K 32
#define SONET_NORMALS_CANONICAL 0
#define SONET_NORMALS_AWAY_FROM_CENTROID 1
#define SONET_NORMALS_TOWARD_VIEWPOINT 2
int sonet_point_knn_f32(const float* data, long long T, int stride, const int64_t* offsets, int S,
                        int K, int32_t* idx, float* dist, sonet_stream_t stream);
long long sonet_point_normals_scratch_bytes(int S);
int sonet_point_normals_f32(const float* data, long long T, int stride, const int64_t* offsets,
                            int S, const int32_t* idx, int K, int orient, const float* view,
                            void* scratch, long long scratch_bytes, float* normals,
                            int normal_stride, float* curvature, sonet_stream_t stream);

/* sonet_point_normals_orient_f32: makes existing normals (estimated, scanned, any) consistently
 * oriented within each cloud by propagating their signs along a minimum spanning tree of the k-NN
 * graph (Hoppe et al. 1992). It changes only signs, in place at normals + row * normal_stride.
 *   Clouds: row g belongs to the cloud ragged_find (csrc/common.cuh) picks over the clamped offsets
 *     when it lies in that cloud's clamped range, to no cloud otherwise, so every row has at most one
 *     cloud even when offsets overlap. Rows of a cloud at a cloud-local index >= max_points are not
 *     vertices: max_points fixes the round schedule without a host synchronisation, and callers pass
 *     the largest cloud size.
 *   Vertices: rows with finite xyz and a finite, non-zero normal. Edges: for each vertex u and each
 *     entry j of idx[u, 0..K) (cloud-local, as sonet_point_knn_f32 writes) in [0, P) with j != u
 *     whose row is a vertex of u's cloud, the undirected edge {u, j}; an edge listed from both ends
 *     is one edge. Its dot = (nx_u*nx_v + ny_u*ny_v) + nz_u*nz_v in fp64, explicitly rounded, its
 *     weight w = fp32(1 - |dot|) rounded once. Edges are ordered strictly by (w, min(u,v), max(u,v))
 *     (cloud-local), so every connected component has exactly one minimum spanning tree.
 *   Anchor: one vertex per component, the codes of sonet_point_normals_f32:
 *     SONET_NORMALS_AWAY_FROM_CENTROID  the vertex farthest from the cloud's centroid (computed as
 *                                       sonet_point_normals_f32 does, over every row of the clamped
 *                                       range), ref = p - c;
 *     SONET_NORMALS_TOWARD_VIEWPOINT    the vertex nearest view[s], ref = view[s] - p;
 *     squared distances ((dx*dx + dy*dy) + dz*dz) in fp64, a NaN distance last, the lowest
 *     cloud-local index on ties. The anchor flips iff dot(n, ref) < 0 in fp64 ((nx*rx + ny*ry) +
 *     nz*rz); a dot of 0 or NaN keeps its input sign. Any other code (CANONICAL too) is refused.
 *   Signs: a vertex is negated iff the anchor's flip XOR the parity of the dot < 0 edges on its tree
 *     path from the anchor is 1. Output normals are exactly +-input; non-vertices are untouched.
 *     Input signs matter only through edges whose dot is exactly 0 and anchors whose dot is 0 or NaN.
 *     component [T] i32 (nullable): the cloud-local index of the vertex's anchor, -1 for every row
 *     that is not a vertex.
 * Limits: every component is anchored on its own; a k-NN graph that bridges two close sheets can
 * carry a flip across them; no edges beyond the k-NN graph are added. max_points must be below
 * SONET_POINT_ORIENT_MAX_POINTS = 2^24 (the pairs are packed as two 24-bit local indices), a
 * narrower limit than sonet_point_knn_f32's.
 * Work: one optional centroid launch, one init launch, 5 launches per round for
 * ceil(log2(max_points)) rounds (a round after one that merged nothing exits at once), then 3.
 * Scratch: sonet_point_normals_orient_scratch_bytes(T, S) bytes of 256-byte aligned device memory
 * (0 for S = 0, where scratch may be null; -1 for T < 0 or S < 0). After a call its first
 * SONET_POINT_ORIENT_MAX_ROUNDS int32 hold 1 for each round that merged components.
 * Like the entries above it allocates nothing, does not synchronise, is deterministic and capturable
 * in a CUDA graph; every loop is bounded (rounds by max_points, pointer jumps by max_points steps).
 * It fails with SONET_ERR_BAD_ARG before any CUDA call for S < 0, T < 0, stride < 3,
 * normal_stride < 3, K outside [1, SONET_POINT_KNN_MAX_K], max_points outside [0, 2^24), an
 * unknown anchor code, null offsets or normals, null data or idx with T > 0, a null view with the
 * viewpoint code, or a missing, too small or misaligned scratch; S = 0 then returns without a
 * launch. */
#define SONET_POINT_ORIENT_MAX_POINTS 16777216
#define SONET_POINT_ORIENT_MAX_ROUNDS 24
long long sonet_point_normals_orient_scratch_bytes(long long T, int S);
int sonet_point_normals_orient_f32(const float* data, long long T, int stride, const int64_t* offsets,
                                   int S, int max_points, const int32_t* idx, int K, int anchor,
                                   const float* view, void* scratch, long long scratch_bytes,
                                   float* normals, int normal_stride, int32_t* component,
                                   sonet_stream_t stream);

/* ---- a-4/a-5/a-8/a-9/a-10: point-wise shared MLP layer (1x1 conv + folded BN + ReLU) ---------
 * Replaces EquivariantLayer.forward / MyConv2d(1x1).forward in eval mode
 * (models/layers.py:203-210, 282-296): out[b,co,p] = act(scale[co]*sum_ci W[co,ci]*X[b,ci,p] +
 * shift[co] (+ addend[b,co,gidx[b,p]])), where X is the channel-concatenation of x0 [B,C0,P]
 * and x1 [B,C1,P] (x1 nullable with C1=0) — the concat of PointResNet (layers.py:431) and of
 * final_pointnet's input (networks.py:192) without materialising it.
 * Wt [C0+C1, Cout] row-major = the conv weight TRANSPOSED (so that a K-slab of weights is
 * contiguous along Cout), packed once by the host; scale/shift [Cout] hold conv bias and
 * eval-mode BatchNorm folded by the host (scale nullable = 1; the host may also fold scale into
 * Wt). relu: activation code (SONET_ACT_NONE / _RELU / _ELU).
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
/* The same loss over whole shapes of any size (losses.seg_loss_ragged, INTEGRATION.md "Whole
 * clouds: the segmenter"): score [T,C] f32 point-major, target [T] int64, cloud b is rows
 * offsets[b] .. offsets[b+1] (offsets [B+1] int64 on the device, offsets_host the same values in
 * host memory). loss: one float, the mean over every counted point of the batch (the rule of
 * sonet_seg_loss_f32 with size_average=1: with equal sizes P it is that entry's bits on the scores
 * laid out [B,C,P]); loss_array [B]: each cloud's own mean. Targets equal to -100 do not count; any
 * other out-of-range target makes its cloud's mean and loss NaN, and no other cloud's; a cloud with
 * no counted point has NaN in loss_array (0/0) and adds nothing to loss. Deterministic: fixed-order
 * fp64 sums of 256-point tile partials. scratch: sonet_seg_loss_ragged_scratch_bytes(B, T) bytes of
 * device memory; it also receives the clouds' tile-start prefix sums from the host (one pageable
 * copy on the stream). Refused before any launch: B < 1, C < 1, T < 0, a null pointer,
 * offsets_host not running from 0 to T without decreasing, a cloud of 2^31 - 256 points or more, 2^31
 * partials or more. Device offsets that disagree with offsets_host are clamped into [0,T] (results
 * unspecified, nothing out of range). No allocation, no host synchronisation. */
long long sonet_seg_loss_ragged_scratch_bytes(int B, long long T);
int sonet_seg_loss_ragged_f32(const float* score, const long long* target, const long long* offsets,
                              const long long* offsets_host, int B, int C, long long T, void* scratch,
                              float* loss, float* loss_array, sonet_stream_t stream);

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
/* Ragged twin over every point of each shape: score [T,C] f32 point-major, seg [T] int64, label [B]
 * int64, offsets [B+1] int64 (shape b owns points offsets[b] .. offsets[b+1]); the same argmax and
 * per-part rule, one launch. pred [T] int64 and correct [B] int32 nullable. The device entry reads
 * offsets on the device only: a shape whose offsets are out of order or outside [0,T] yields
 * iou_shape[b] = NaN, as does a label outside the table. */
int sonet_seg_iou_ragged_f32(const float* score, const long long* seg, const long long* label,
                             const long long* offsets, int B, int C, long long T,
                             const int32_t* part_offsets, const int32_t* part_ids, int num_categories,
                             double* iou_shape, long long* pred, int32_t* correct, sonet_stream_t stream);
/* The same over host pointers; validates offsets (0 .. T, non-decreasing), the table and every
 * label: SONET_ERR_BAD_ARG otherwise. */
int sonet_seg_iou_ragged_cpu_f32(const float* score, const long long* seg, const long long* label,
                                 const long long* offsets, int B, int C, long long T,
                                 const int32_t* part_offsets, const int32_t* part_ids,
                                 int num_categories, double* iou_shape, long long* pred,
                                 int32_t* correct, int thread_num);

/* SOM assignment and decentring of one chunk of a ragged point set for the segmenter's per-point
 * head (segmenter.Model.score_points). points [total,6] f32 (xyz | normal), offsets [B+1] int64
 * (device; cloud b owns rows offsets[b] .. offsets[b+1]), node [B,3,M] the loader's SOM nodes,
 * cluster_mean [B,3,M] the encoder's centres of the sampled forward. Rows [row0, row0+rows) find their
 * k nearest nodes of their cloud with sonet_som_assign's arithmetic and tie rule and are written
 * copy-major over k*rows_pad columns (column s*rows_pad + r: copy s of row r): gidx [k*rows_pad]
 * int32 = b*M + node (a flat index into the node-level addend laid out [C, B*M]); x_aug
 * [3(+3), k*rows_pad] = xyz - centre (| normal); pt [9(+3), k*rows_pad] = x_dec | xyz | centre
 * (| normal). with_sn: 1 writes the normal channels. Columns of rows >= rows are zero, node 0.
 * 1 <= M <= 256, 1 <= k <= min(4, M), rows <= rows_pad, row0 + rows <= total. offsets are not read
 * on the host (the caller validates them); one launch. */
int sonet_seg_points_assign_f32(const float* points, long long total, const long long* offsets, int B,
                                const float* node, const float* cluster_mean, int M, int k, int with_sn,
                                long long row0, int rows, int rows_pad, int32_t* gidx, float* x_aug,
                                float* pt, sonet_stream_t stream);

/* ---- whole clouds of any size: the encoder's stage before the first per-node max, ragged ---------
 * (networks.Encoder.forward_ragged, csrc/som_ragged.cu, INTEGRATION.md "Whole clouds of any size").
 * points [T,6] f32 (xyz | normal), offsets [B+1] int64 (device): cloud b is rows offsets[b] ..
 * offsets[b+1], P_b points. Its k stacked copies are the columns k*offsets[b] + s*P_b + n (copy s of
 * point n, the reference's x_stack order at N = P_b), k*T columns in all. node [B,3,M] the loader's
 * SOM nodes. Every offset is clamped to [0,T] and a decreasing pair is an empty cloud, so no input
 * reads or writes out of range (the results of such offsets are unspecified; callers validate them).
 * Limits: 1 <= M <= 256, 1 <= k <= min(4, M), k*T < 2^31, B*M < 2^31; no scratch.
 *   assign: min_idx [k*T] i32 = the cloud-local node of every copy (sonet_som_assign's arithmetic
 *     and tie rule against node[b]), count [B,M] i32, row_max [B,M] i32 = count > 0. Two memsets and
 *     one launch, a thread per point.
 *   group_decenter: CTA per cloud, any P_b (the stable sort runs through global memory), T < 2^24.
 *     cluster_mean [B,3,M] = sum / (count + 1e-5), the sums in sonet_som_group_decenter's order (a
 *     node's copies in ascending stacked order, lane l of a warp sums copies l, l+32, ... in groups of
 *     four, xor butterfly 16..1), so a cloud gets that entry's bits at N = P_b; x_sorted [3|6, k*T]
 *     (row stride k*T) the decentred copies (| normals, with_sn = 1) grouped by (cloud, node),
 *     ascending stacked order inside a node, cloud b's block at its own columns; node_sorted [k*T]
 *     i32 = b*M + m; pos0 [B] i32 = the sorted column of cloud b's copy 0.
 *   decenter: x_aug [3|6, k*T] = the decentred copies in stacked order (the unfused route).
 *   sonet_pointresnet_tc_pool_ragged_forward: sonet_pointresnet_tc_pool_forward_act over x_sorted
 *     [Cin, P] as ONE batch row (P = k*T) with node_sorted's flat ids (grouped, each < B*M): the max of
 *     every (cloud, channel, node) goes to pool_keys [B,384,M] (sonet_pool_keys_init's value on
 *     entry), the features of the row pos0[b] to p0 [b,384]; act = SONET_ACT_RELU or _ELU, f16 != 0
 *     the one-product mode. sonet_pool_finalize / sonet_knn_assemble_pool_f32 read the keys as usual.
 *   sonet_index_max_ragged_f32: data [C, ld] (ld >= k*T) in stacked column order, index the
 *     min_idx above -> out_idx [B,C,M] i32 (cloud-local stacked column, the lowest on ties) and
 *     out_val [B,C,M] f32 (nullable): index_max's semantics per cloud at N = k*P_b (max > -1000,
 *     else column 0 and the value of the cloud's copy 0; NaN never a maximum). C <= 65535*16.
 * All deterministic; no allocation, no host synchronisation. */
int sonet_som_assign_ragged_f32(const float* points, long long T, const long long* offsets, int B,
                                const float* node, int M, int k, int32_t* min_idx, int32_t* count,
                                int32_t* row_max, sonet_stream_t stream);
int sonet_som_group_decenter_ragged_f32(const float* points, long long T, const long long* offsets,
                                        int B, int M, int k, int with_sn, const int32_t* min_idx,
                                        float* cluster_mean, float* x_sorted, int32_t* node_sorted,
                                        int32_t* pos0, sonet_stream_t stream);
int sonet_som_decenter_ragged_f32(const float* points, long long T, const long long* offsets, int B,
                                  int M, int k, int with_sn, const int32_t* min_idx,
                                  const float* cluster_mean, float* x_aug, sonet_stream_t stream);
int sonet_pointresnet_tc_pool_ragged_forward(const float* x_sorted, int Cin, int P, const void* blob,
                                             const float* fparams, const int32_t* node_sorted,
                                             const int32_t* pos0, int B, int M, int act, int f16,
                                             int32_t* pool_keys, float* p0, sonet_stream_t stream);
int sonet_index_max_ragged_f32(const float* data, int C, long long ld, const int32_t* index,
                               const long long* offsets, int B, long long T, int M, int k,
                               int32_t* out_idx, float* out_val, sonet_stream_t stream);

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
 * A point with no finite nearest neighbour (its minimum squared distance over non-NaN candidates
 * is +inf, or it has no non-NaN candidate) gets index 0 and the element of the pair (point, other
 * cloud's point 0): NaN if either has a NaN, +inf on overflow. Indices are always in range.
 * All reductions run in a fixed order (bit-reproducible). */
int sonet_chamfer_f32(const float* pred, const float* gt, int B, int Mp, int N, int32_t* idx_fwd,
                      int32_t* idx_bwd, float* elem_fwd, float* elem_bwd, float* loss_fwd_arr,
                      float* loss_bwd_arr, float* loss, sonet_stream_t stream);
/* The same against whole ground-truth clouds of any size (losses.chamfer_ragged, INTEGRATION.md
 * "Whole clouds: the auto-encoder"): pred [B,3,Mp]; points [T,ld] f32 rows (xyz first, ld >= 3;
 * DeviceDataset's [T,6]), cloud b is rows offsets[b] .. offsets[b+1] (P_b points; offsets [B+1]
 * int64 on the device, offsets_host the same values in host memory). Outputs as sonet_chamfer_f32
 * with the gt side ragged: idx_fwd [B,Mp] (cloud-local rows) and idx_bwd [T] (nullable, together),
 * elem_fwd [B,Mp], elem_bwd [T], loss_fwd_arr / loss_bwd_arr [B], loss [3]. Cloud b's entries are
 * sonet_chamfer_f32's bits for that cloud alone at N = P_b (same arithmetic, tie rule, non-finite
 * rule and summation order); loss is the mean over clouds of the per-cloud means, so every cloud
 * counts once in backward_loss whatever its size. tile_start: device scratch of B+1 int32, written
 * from the host (one pageable copy on the stream) with the prefix sums of the clouds' 1024-column
 * tiles. Refused before any launch: B < 1, Mp < 1, ld < 3, a null pointer, idx_fwd without idx_bwd
 * or the reverse, offsets_host not running from 0 to T, an empty cloud, a cloud of 2^24 points or
 * more. Device offsets that disagree with offsets_host are clamped into [0,T] (results unspecified,
 * nothing out of range). Deterministic; no allocation, no host synchronisation. */
int sonet_chamfer_ragged_f32(const float* pred, int B, int Mp, const float* points, long long T,
                             long long ld, const long long* offsets, const long long* offsets_host,
                             int32_t* tile_start, int32_t* idx_fwd, int32_t* idx_bwd, float* elem_fwd,
                             float* elem_bwd, float* loss_fwd_arr, float* loss_bwd_arr, float* loss,
                             sonet_stream_t stream);

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
 *     (Wt, scale); relu is the activation code, here and in the _rows, _grouped, _dev and _f16
 *     entries (ELU in fp32 after the GEMM, in every precision mode).
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

/* ---- the point-wise layer at node-level row counts, csrc/nodegemm_tc.cu ------------------------
 * The same layer, bit for bit, with the activations pre-split into fp16 hi/lo operand images in
 * global memory so that both wgmma operands arrive by bulk copy (the encoder's final PointNet:
 * two layers over B*M rows, where the generic kernel's per-chunk conversion dominates).
 *   image_bytes(rows, C, f16): size of the images of a [rows x C] activation matrix (16-byte
 *     aligned device memory); f16 != 0: the hi image only, for the one-product fp16 mode.
 *   split_pack (device pointers): cat(x0 [B,C0,P], x1 [B,C1,P] or NULL) -> img.
 *   forward (device pointers): img (of B*P rows x Cin) x the blob of sonet_pointwise_tc_pack
 *     -> act(inv_scale * GEMM + shift), written either as out [B,Cout,P] fp32 (img_out NULL), the
 *     values sonet_pointwise_tc_forward writes, or as img_out (out NULL), the images split_pack
 *     would build from that tensor: the next layer's input. act is the activation code; f16 must
 *     be the value the images were built with (then: the values of sonet_pointwise_tc_forward_f16).
 *   No allocation, no host synchronisation, deterministic, CUDA graph capturable. */
long long sonet_nodegemm_image_bytes(long long rows, int C, int f16);
int sonet_nodegemm_split_pack(const float* x0, int C0, const float* x1, int C1, int B, int P,
                              int f16, void* img, sonet_stream_t stream);
int sonet_nodegemm_tc_forward(const void* img, int Cin, int B, int P, const void* blob,
                              float inv_scale, const float* shift, int Cout, int act, int f16,
                              void* img_out, float* out, sonet_stream_t stream);

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

/* ---- explicit activation of the fused kernels ---------------------------------------------------
 * sonet_pointresnet_tc_forward / _pool_forward and sonet_knn_mlp_tc_forward hard-code ReLU (they
 * equal these entries with act = SONET_ACT_RELU, f16 = 0). These take the activation of the hidden
 * layers (the PointResNet's layers 0-2, both KNN layers): act = SONET_ACT_RELU or SONET_ACT_ELU
 * (anything else, SONET_ACT_NONE included, fails with SONET_ERR_BAD_ARG), and f16 != 0 selects the
 * one-product fp16 mode of the `_f16` entries. Otherwise the arguments, blobs and properties of the
 * entries without the suffix. ELU runs in fp32 in both modes. The PointResNet's per-node pool acts
 * on the bare layer 3 (unaffected), and the KNN kernel's max over the neighbours on the raw
 * accumulators stays exact: ELU is non-decreasing like ReLU (csrc/knn_tc.cu). */
int sonet_pointresnet_tc_forward_act(const float* x, int Cin, int B, int P, const void* blob,
                                     const float* fparams, int act, int f16, float* out,
                                     sonet_stream_t stream);
int sonet_pointresnet_tc_pool_forward_act(const float* x_sorted, int Cin, int B, int P,
                                          const void* blob, const float* fparams,
                                          const int32_t* node_sorted, const int32_t* pos0, int M,
                                          int act, int f16, int32_t* pool_keys, float* p0,
                                          sonet_stream_t stream);
int sonet_knn_mlp_tc_forward_act(const float* coord, const float* center, const int64_t* idx, int B,
                                 int M, int K, int Kstride, const float* Y, long long y_cstride,
                                 long long y_nstride, const float* w1, const void* blob,
                                 float inv_scale, const float* shift2, int act, int f16, float* out,
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
