/*
 * b200gnn.h — C ABI of the H100-native (sm_90a) sparse message-passing engine.
 *
 * This is the drop-in boundary for the hot path of chaitjo/efficient-gnns
 * (SURVEY.md §8b).  The reference reaches its sparse arithmetic through
 * un-vendored Python/C++ dependencies (torch_sparse / torch_scatter / PyG);
 * each entry point below names the reference call site (file:line, relative
 * to the reference repository's root) whose arithmetic it replaces.
 *
 * Conventions
 *   - All pointers are DEVICE pointers unless the name ends in `_host`.
 *   - The library never allocates or frees: callers own every buffer,
 *     including workspaces (size helpers are provided).
 *   - Every call is asynchronous on `stream` (a cudaStream_t passed as void*),
 *     performs no host<->device synchronisation and is safe under CUDA-graph
 *     capture.
 *   - Return value: 0 on success, a negative B200GNN_ERR_* otherwise.
 *     b200gnn_last_cuda_error() gives the CUDA error string of the last
 *     B200GNN_ERR_CUDA on the calling thread.
 *   - Engine-side indices are int32 (the Python host narrows the reference's
 *     int64 once, with a range check); features are fp32 row-major with an
 *     explicit leading dimension (in elements).
 */
#ifndef B200GNN_H_
#define B200GNN_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B200GNN_OK 0
#define B200GNN_ERR_BAD_ARG (-1)
#define B200GNN_ERR_UNSUPPORTED (-2)
#define B200GNN_ERR_CUDA (-3)

#define B200GNN_REDUCE_SUM 0
#define B200GNN_REDUCE_MEAN 1

#define B200GNN_ABI_VERSION 2

int b200gnn_abi_version(void);
const char* b200gnn_error_string(int code);
const char* b200gnn_last_cuda_error(void);
/* Number of kernel launches issued through this library by the calling
 * process since load / since the last reset (bench.py's gpu_launches). */
int64_t b200gnn_launch_count(void);
void b200gnn_reset_launch_count(void);

/* ------------------------------------------------------------------ *
 * CSR chunk plan: load balance for power-law graphs.  Chunk c is the run of
 * consecutive rows starting at the first row r with
 *     rowptr[r] + r*row_cost >= c*chunk_nnz ,
 * so each chunk (= one warp of the SpMM kernel) holds about chunk_nnz
 * non-zeros (+ row_cost per row, which also spreads empty rows).
 *   n_chunks = b200gnn_csr_chunk_count(...)   (host arithmetic only)
 *   chunk_rowptr: int32[n_chunks+1], chunk_rowptr[n_chunks] = n_rows
 * ------------------------------------------------------------------ */
int64_t b200gnn_csr_chunk_count(int64_t n_rows, int64_t nnz, int32_t chunk_nnz,
                                int32_t row_cost);
int b200gnn_csr_chunk_plan(const int32_t* rowptr, int64_t n_rows, int64_t nnz,
                           int32_t chunk_nnz, int32_t row_cost,
                           int32_t* chunk_rowptr, void* stream);

/* ------------------------------------------------------------------ *
 * CSR hub plan.  Rows whose degree exceeds `hub_threshold` are split into
 * segments of `seg_len` non-zeros processed by whole CTAs, so one hub node
 * (ARXIV-shape: degree ~2e4) cannot serialise a warp.  Built once per graph
 * and cached next to rowptr, like torch_sparse's SparseStorage caches
 * rowcount/colptr/csr2csc (used via arxiv_pyg/gnn.py:236-240).
 *   counts_out: int32[2] = {n_hub_rows, n_segments}
 *   hub_rows:   int32[n_hub]  ascending row ids
 *   hub_segptr: int32[n_hub+1] exclusive prefix of per-row segment counts
 * ------------------------------------------------------------------ */
int b200gnn_csr_hub_count(const int32_t* rowptr, int64_t n_rows,
                          int32_t hub_threshold, int32_t seg_len,
                          int32_t* counts_out, void* stream);
int b200gnn_csr_hub_fill(const int32_t* rowptr, int64_t n_rows,
                         int32_t hub_threshold, int32_t seg_len,
                         int32_t* hub_rows, int32_t* hub_segptr,
                         int64_t n_hub, void* stream);

/* ------------------------------------------------------------------ *
 * Row-segmented CSR SpMM  Y[i,:] = reduce_{e in row i} val[e] * X[col[e],:]
 * Replaces torch_sparse spmm_sum / spmm_mean reached from
 *   GCNConv  arxiv_pyg/gnn.py:47,52   (reduce=sum, weighted)
 *   SAGEConv arxiv_pyg/gnn.py:79,84   (reduce=mean, val==NULL)
 *   adj_t.matmul(x, reduce='mean')  mag_pyg/gnn.py:162
 * and their backward (the same kernel on the CSC view).
 *   val  : NULL => all ones.
 *   bias : NULL or float[K]; added after the reduction (GCNConv `out += bias`).
 *   stat_partial : NULL or float[b200gnn_spmm_stat_slots()][2][K]; every slot
 *          receives a deterministic partial column sum (slot,0,:) and sum of
 *          squares (slot,1,:) of the rows of Y it produced, for the
 *          BatchNorm1d that follows the conv (arxiv_pyg/gnn.py:48).
 *   chunk_rowptr/n_chunks : plan from b200gnn_csr_chunk_plan (required).
 *   hub_* : plan from b200gnn_csr_hub_*; n_hub==0 disables the split path
 *          (then hub_threshold must be >= the maximum degree or INT32_MAX).
 *   hub_workspace : float[n_seg][K] scratch for segment partials.
 * MEAN divides by max(degree,1); empty rows give 0 (+bias).
 * ------------------------------------------------------------------ */
int64_t b200gnn_spmm_stat_slots(int64_t n_chunks, int64_t n_hub);
/* Kernel selection for tuning / A-B measurement: 0 = automatic (cp.async-pipelined kernel for K in
 * {128,256,512}, multi-row kernel for K <= 64, register-staged kernel otherwise), 1 = always the
 * register-staged kernel. */
void b200gnn_spmm_set_variant(int variant);
int b200gnn_spmm_csr_f32(const int32_t* rowptr, const int32_t* col,
                         const float* val, const float* X, int64_t ldx,
                         float* Y, int64_t ldy, int64_t n_rows, int64_t n_src,
                         int64_t K, int reduce, const float* bias,
                         float* stat_partial, const int32_t* chunk_rowptr,
                         int64_t n_chunks, int32_t hub_threshold,
                         int32_t seg_len, const int32_t* hub_rows,
                         const int32_t* hub_segptr, int64_t n_hub,
                         int64_t n_seg, float* hub_workspace, void* stream);
/* The same product with the C->R layout exchange of the multi-GPU engine fused into the epilogue: output row i is stored to
 * Y_ptrs[q][(i - row_off[q]) * ldy_dst + col_dst ...] for the rank q that owns it (HOST arrays: `world` peer-mapped device
 * pointers, world+1 ascending row offsets).  Supported where the TMA kernels (K % 128 == 0) or the narrow kernel (K <= 64,
 * no fused statistics) run, else B200GNN_ERR_UNSUPPORTED. */
int b200gnn_spmm_csr_scatter_f32(const int32_t* rowptr, const int32_t* col, const float* val, const float* X,
                                 int64_t ldx, float* const* Y_ptrs, const int32_t* row_off, int32_t world,
                                 int64_t ldy_dst, int64_t col_dst, int64_t n_rows, int64_t n_src, int64_t K,
                                 int reduce, const float* bias, const int32_t* chunk_rowptr, int64_t n_chunks,
                                 int32_t hub_threshold, int32_t seg_len, const int32_t* hub_rows,
                                 const int32_t* hub_segptr, int64_t n_hub, int64_t n_seg,
                                 float* hub_workspace, void* stream);

/* ------------------------------------------------------------------ *
 * Dense row-major [n_rows,K] passes between the aggregations of a layer:
 * BatchNorm1d(train) -> ReLU -> dropout (arxiv_pyg/gnn.py:48-50) and their
 * backward.  K % 4 == 0, K <= 1024, 16-byte aligned, contiguous (ld == K).
 * All reductions go through `partial[slots][2][K]` scratch with
 * slots = b200gnn_rows_slots(n_rows) (one CTA per slot, fixed order =>
 * deterministic).
 * ------------------------------------------------------------------ */
int64_t b200gnn_rows_slots(int64_t n_rows);
/* partial[s][0][:] = column sums, partial[s][1][:] = column sums of squares */
int b200gnn_col_stats_f32(const float* Y, int64_t n_rows, int64_t K,
                          float* partial, int64_t slots, void* stream);
/* out[K] = column sums of Y (bias gradient of the last conv) */
int b200gnn_col_sum_f32(const float* Y, int64_t n_rows, int64_t K, float* out,
                        float* partial, int64_t slots, void* stream);
/* partials (from the SpMM epilogue or col_stats) -> batch mean / invstd and the
 * fused affine  scale = gamma*invstd, shift = beta - mean*scale ; running
 * statistics updated like nn.BatchNorm1d (momentum, unbiased variance) unless
 * running_mean/running_var are NULL. */
int b200gnn_bn_finalize_f32(const float* partial, int64_t slots, int64_t K,
                            int64_t n_rows, const float* gamma,
                            const float* beta, float eps, float momentum,
                            float* running_mean, float* running_var,
                            float* mean_out, float* invstd_out,
                            float* scale_out, float* shift_out, void* stream);
/* out = dropout_p(relu(Y*scale + shift)); scale/shift NULL => identity affine;
 * relu: 0/1.  The keep-mask is a pure function of (seed, effective offset,
 * element index) (Philox4x32-10) with
 *     effective offset = offset + (step_dev ? *step_dev * step_mul : 0),
 * step_dev being a device int32 (e.g. the Adam step counter) so a captured
 * CUDA graph draws a fresh mask on every replay;
 * row_offset: global index of row 0 of Y (node-parallel shards draw the mask
 * of their own rows of the global matrix; 0 on a single GPU);
 * b200gnn_dropout_mask_u8 materialises the mask of a given effective offset.
 * Uniforms: when p*65536 is integral (the reference's p = 0.5) eight 16-bit
 * uniforms per Philox block, keep iff u16 >= p*65536 (exact); otherwise four
 * 24-bit uniforms per block, keep iff u >= p. */
int b200gnn_affine_relu_dropout_f32(const float* Y, float* out, int64_t n_rows,
                                    int64_t K, const float* scale,
                                    const float* shift, int relu, float p,
                                    uint64_t seed, uint64_t offset,
                                    const int32_t* step_dev, uint64_t step_mul,
                                    uint64_t row_offset, void* stream);
/* Block form (node-parallel engine, SURVEY.md §8e "identical dropout masks by global node id"): local row r is node
 * rowmap[r] (or r + row_offset when rowmap is NULL), local columns are [col_offset, col_offset + K) of a
 * K_global-wide matrix; every keep decision equals the one the full-matrix call takes for that (node, feature). */
int b200gnn_affine_relu_dropout_mapped_f32(const float* Y, float* out, int64_t n_rows, int64_t K,
                                           const float* scale, const float* shift, int relu, float p,
                                           uint64_t seed, uint64_t offset, const int32_t* step_dev,
                                           uint64_t step_mul, const int32_t* rowmap, uint64_t row_offset,
                                           int64_t K_global, int64_t col_offset, void* stream);
/* ... with the C->R layout exchange fused: every output row is ALSO stored to the R-layout buffer of the rank owning the node:
 * dst_ptrs[q] + (r - row_off[q]) * ld_dst + col_offset (HOST arrays of `world` peer-mapped device pointers / world+1 offsets). */
int b200gnn_affine_relu_dropout_scatter_f32(const float* Y, float* out, int64_t n_rows, int64_t K,
                                            const float* scale, const float* shift, int relu, float p,
                                            uint64_t seed, uint64_t offset, const int32_t* step_dev,
                                            uint64_t step_mul, const int32_t* rowmap, uint64_t row_offset,
                                            int64_t K_global, int64_t col_offset, float* const* dst_ptrs,
                                            const int32_t* row_off, int32_t world, int64_t ld_dst, void* stream);
int b200gnn_dropout_mask_u8(uint8_t* mask, int64_t n_rows, int64_t K, float p,
                            uint64_t seed, uint64_t offset, void* stream);
/* b200gnn_dropout_mask_u8 of the effective offset offset + *step_dev * step_mul, read on the device: the edge keep-mask of
 * the GAT step's edge drop (arxiv_dgl/models.py:207-212), fresh on every replay of a captured graph. */
int b200gnn_dropout_mask_step_u8(uint8_t* mask, int64_t n_rows, int64_t K, float p, uint64_t seed, uint64_t offset,
                                 const int32_t* step_dev, uint64_t step_mul, void* stream);
/* The keep decisions of b200gnn_affine_relu_dropout_f32 (row_offset 0) packed one bit per element, for n_layers
 * [n_rows, K] activations in one launch: layer l uses effective offset offset + l (+ *step_dev * step_mul) and fills
 * bits[l][row][w], w < ceil(K/32), bit b = column 32 w + b (bits past K are zero).  Needs no input: it can run next to
 * whatever precedes the first consumer.  The fused GEMMs (_act / _bits entry points) recompute the activation from Y,
 * scale / shift and these bits; b200gnn_affine_relu_bits_f32 materialises it (bit-identical to
 * b200gnn_affine_relu_dropout_f32 with relu = 1 for the same decisions). */
int b200gnn_dropout_bits_u32(uint32_t* bits, int64_t n_layers, int64_t n_rows, int64_t K, float p, uint64_t seed,
                             uint64_t offset, const int32_t* step_dev, uint64_t step_mul, void* stream);
int b200gnn_affine_relu_bits_f32(const float* Y, const uint32_t* bits, const float* scale, const float* shift,
                                 float p, float* out, int64_t n_rows, int64_t K, void* stream);
/* out[i] = row idx[i] (int64) of a hidden activation, [n_idx, K] contiguous: X[idx[i]] (row pitch ldx), or, with bits
 * (uint32 [rows][ceil(K/32)] of b200gnn_dropout_bits_u32), dropout(relu(X[idx[i]] * scale + shift)) formed exactly as
 * b200gnn_affine_relu_bits_f32 forms it (bit-identical).  The G-CRD step's model.out_feat[train_idx]
 * (arxiv_pyg/gnn.py:296) without the [N, K] activation. */
int b200gnn_gather_rows_act_f32(const float* X, int64_t ldx, const int64_t* idx, int64_t n_idx, int64_t K,
                                const uint32_t* bits, const float* scale, const float* shift, float p, float* out,
                                void* stream);
/* Backward of out = dropout_p(relu(Y)) (no BatchNorm): dY = dOut * [Xout > 0] / (1-p), contiguous [n_rows, K]
 * rows, K a multiple of 4; dY may alias dOut. */
int b200gnn_relu_dropout_bwd_f32(const float* dOut, const float* Xout, float* dY,
                                 int64_t n_rows, int64_t K, float p, void* stream);
/* Backward of out = dropout_p(relu(BN_train(Y))): given dOut, out (for the
 * mask: out>0 <=> kept and active), Y and the saved batch mean/invstd, writes
 * dY, dgamma[K], dbeta[K] and (if non-NULL) dbias[K] = column sums of dY.
 * coef: float[3*K] scratch.  dY must not alias dOut. */
int b200gnn_bn_act_bwd_f32(const float* dOut, const float* Xout, const float* Y,
                           const float* mean, const float* invstd,
                           const float* gamma, int64_t n_rows, int64_t K,
                           float p, float* dY, float* dgamma, float* dbeta,
                           float* dbias, float* partial, int64_t slots,
                           float* coef, void* stream);
/* The same backward in two phases, for node-parallel runs that all-reduce the
 * column sums between them: reduce -> partial[slots][2][K];  apply consumes
 * `sums[sum_slots][2][K]` (the local partials, or ONE slot of cross-rank sums)
 * with n_norm = global row count. */
int b200gnn_bn_act_bwd_reduce_f32(const float* dOut, const float* Xout,
                                  const float* Y, const float* mean,
                                  const float* invstd, int64_t n_rows,
                                  int64_t K, float p, float* partial,
                                  int64_t slots, void* stream);
int b200gnn_bn_act_bwd_apply_f32(const float* dOut, const float* Xout,
                                 const float* Y, const float* mean,
                                 const float* invstd, const float* gamma,
                                 const float* sums, int64_t sum_slots,
                                 int64_t n_norm, int64_t n_rows, int64_t K,
                                 float p, float* dY, float* dgamma,
                                 float* dbeta, float* dbias, float* partial,
                                 int64_t slots, float* coef, void* stream);
/* Xout == NULL in b200gnn_bn_act_bwd_apply_f32: dOut already holds
 * dz = dOut * [Xout > 0] / (1-p), as stored by b200gnn_gemm_tf32x3_bnbwd_f32
 * (whose partial buffer is then `sums`); dY may alias dOut. */
/* out[K2] = sum over slots of partial[slot][K2] (K2 = 2*K for statistics) */
int b200gnn_partial_reduce_f32(const float* partial, int64_t slots, int64_t K2,
                               float* out, void* stream);
/* torch.optim.Adam (defaults: no amsgrad, no weight decay) over flat buffers;
 * *step (device int32) is the number of steps already taken and is incremented
 * (arxiv_pyg/gnn.py:192-193, 308-315). */
int b200gnn_adam_step_f32(float* params, const float* grads, float* exp_avg,
                          float* exp_avg_sq, int64_t n, float lr, float beta1,
                          float beta2, float eps, int32_t* step, void* stream);
/* torch.optim.RMSprop(lr, alpha, eps, weight_decay) without momentum or centring over flat buffers, with the linear warm-up
 * of arxiv_dgl/gat.py:110-113: the rate of the step is lr * min(*step + 1, warmup) / warmup, formed in double and rounded
 * once (warmup = 0: lr).  *step (device int32, steps already taken) is incremented.  An entry with zero parameter and
 * gradient keeps zero parameter and square_avg. */
int b200gnn_rmsprop_step_f32(float* params, const float* grads, float* square_avg, int64_t n, double lr, int64_t warmup,
                             double alpha, double eps, double weight_decay, int32_t* step, void* stream);

/* ------------------------------------------------------------------ *
 * The training recipe of the arxiv GAT teacher (arxiv_dgl/gat.py:98-183).  Every call is graph-capturable: the step
 * counter, the loss-row count and the best loss are read on the device.
 * role (uint8[n_rows]): 0 none, 1 input (a training row whose label is an input, or without labels a training row outside
 * the loss), 2 pred (a training row the loss runs on), 3 val / test.
 * cnt_part: int32[b200gnn_teacher_slots(n_rows)], the per-CTA count of role-2 rows.
 * partial: double[6 * b200gnn_teacher_slots(rows visited)] scratch.  C <= 256.
 * ------------------------------------------------------------------ */
int64_t b200gnn_teacher_slots(int64_t n_items);
/* Roles and the label block X[:, col0 : col0 + C] of every row: one-hot labels[r] for role-1 rows when C > 0, zero for
 * every other row.  row_pos[r]: position in train_idx (>= 0), -1 for val / test, -2 otherwise.  Training (eval == 0):
 * training position j is masked iff b200gnn_dropout_mask_u8 at p = mask_rate drops flat element j for the offset
 * offset + *step_dev * step_mul; masked rows are the label rows (use_labels) or the loss rows (no labels).  eval != 0:
 * every training row is a label row and nothing is drawn (step_dev may be NULL).  mask_in (uint8[n_train], optional)
 * replaces the draw with a given mask, e.g. a recorded torch.rand draw. */
int b200gnn_label_inputs_f32(float* X, int64_t ldx, int64_t col0, int64_t C, int64_t n_rows, const int32_t* row_pos,
                             const int64_t* labels, int eval, float mask_rate, uint64_t seed, uint64_t offset,
                             const int32_t* step_dev, uint64_t step_mul, const uint8_t* mask_in, int use_labels, uint8_t* role,
                             int32_t* cnt_part, void* stream);
/* out[r, 0:C] = softmax(logits[r, 0:C]) for every row with bit role[r] set in role_mask (every row when role is NULL). */
int b200gnn_label_softmax_f32(const float* logits, int64_t ld, int64_t C, int64_t n_rows, const uint8_t* role, int role_mask,
                              float* out, int64_t ldo, void* stream);
/* custom_loss_function (gat.py:98-101) over the role-2 rows of train_idx: loss_out[0] = mean(log(eps + CE_i) - log eps),
 * eps = 1 - ln 2, normalised by the device count of role-2 rows; dlogits of those rows = (softmax - onehot) /
 * ((eps + CE_i) * n) (the caller zeroes the rest); acc_out[0] = first-maximum argmax accuracy over all of train_idx. */
int b200gnn_logce_fwd_bwd_f32(const float* logits, int64_t ld, int64_t C, const int64_t* train_idx, int64_t n_train,
                              const int64_t* labels, const uint8_t* role, const int32_t* cnt_part, int64_t n_cnt,
                              float* dlogits, int64_t ldd, float* loss_out, float* acc_out, double* partial, void* stream);
/* evaluate()'s losses and accuracies (gat.py:168-183): idx = [train | val | test] (sizes n0, n1, n2);
 * loss_out[s] = custom_loss_function, acc_out[s] = first-maximum argmax accuracy of split s. */
int b200gnn_split_eval_f32(const float* logits, int64_t ld, int64_t C, const int64_t* idx, int64_t n0, int64_t n1, int64_t n2,
                           const int64_t* labels, float* loss_out, float* acc_out, double* partial, void* stream);
/* The best-epoch snapshot (gat.py:217-222): if *cand < *best (never for NaN), dst_i = src_i (n_i floats, a multiple of 4,
 * 16-byte aligned; n_i = 0 skips), then *best = *cand. */
int b200gnn_snapshot_if_better_f32(const float* cand, float* best, const float* src0, float* dst0, int64_t n0,
                                   const float* src1, float* dst1, int64_t n1, const float* src2, float* dst2, int64_t n2,
                                   void* stream);

/* ------------------------------------------------------------------ *
 * Row-wise classification / logit-KD loss with its gradient in one pass.
 *   kd_criterion(logits[train_idx], labels[train_idx], teacher[train_idx],
 *                alpha, T)                  arxiv_pyg/criterion.py:8-21
 *   F.cross_entropy(out, labels)            arxiv_pyg/gnn.py:112  (teacher_logits == NULL)
 * logits / teacher_logits / dlogits are FULL [N,C] matrices (leading dims ld/ldt/ldd);
 * train_idx (int64[n_train], NULL => rows 0..n_train-1) selects the rows, labels is the
 * full int64[N] vector.  dlogits rows in train_idx receive d loss / d logits; the caller
 * zeroes the other rows.  loss_out[3] = {loss, loss_cls, loss_kd}.
 * n_norm: row count the means are taken over (0 => n_train; node-parallel
 * shards pass the GLOBAL number of training rows and sum loss_out across ranks).
 * partial: float[2*b200gnn_kd_partials(n_train)] scratch.  C <= 1024 (ogbn-mag: 349).
 * ------------------------------------------------------------------ */
int64_t b200gnn_kd_partials(int64_t n_train);
int b200gnn_kd_loss_fwd_bwd_f32(const float* logits, int64_t ld,
                                const int64_t* train_idx, int64_t n_train,
                                const int64_t* labels,
                                const float* teacher_logits, int64_t ldt,
                                int64_t C, float alpha, float T,
                                int64_t n_norm, float* dlogits, int64_t ldd,
                                float* loss_out, float* partial, void* stream);

/* ------------------------------------------------------------------ *
 * fp32-faithful dense GEMM on the Hopper tensor cores (wgmma, 3xTF32 split,
 * fp32 accumulation in registers):   C[M,N] = A[M,K] * B[N,K]^T (+ bias[N])
 * Replaces the fp32 cuBLAS contractions behind GCNConv's `x @ weight`,
 * nn.Linear and their input gradients (arxiv_pyg/gnn.py:47,52,79,84 via PyG).
 *   A    : fp32, row-major, split into tf32 hi/lo on the fly inside the kernel.
 *   B_hi, B_lo : the [N,K] operand pre-split by b200gnn_split_tf32_f32
 *          (weights are tiny; `transpose` lets [K,N] storage feed it).
 * lda/ldb multiples of 4 floats, 16-byte aligned bases (TMA); any M, N, K.
 * Dropped terms are O(2^-22) relative, i.e. within the 1e-5 parity budget.
 * ------------------------------------------------------------------ */
int b200gnn_split_tf32_f32(const float* W, int64_t rows, int64_t cols,
                           int transpose, float* hi, float* lo, void* stream);
int b200gnn_gemm_tf32x3_f32(const float* A, int64_t lda, const float* B_hi,
                            const float* B_lo, int64_t ldb, float* C,
                            int64_t ldc, int64_t M, int64_t N, int64_t K,
                            const float* bias, void* stream);
/* C += A · B^T (accumulating epilogue; same operands as above, no bias). */
int b200gnn_gemm_tf32x3_acc_f32(const float* A, int64_t lda, const float* B_hi, const float* B_lo,
                                int64_t ldb, float* C, int64_t ldc, int64_t M, int64_t N, int64_t K,
                                void* stream);
/* C[row_idx[m]] = (A · B^T)[m]: row-indexed stores (row_idx int64, distinct); C rows not named are untouched.  The G-CRD
 * student head's input gradient stored into the training rows of d out_feat (arxiv_pyg/gnn.py:296). */
int b200gnn_gemm_tf32x3_rowidx_f32(const float* A, int64_t lda, const float* B_hi, const float* B_lo,
                                   int64_t ldb, float* C, int64_t ldc, int64_t M, int64_t N, int64_t K,
                                   const int64_t* row_idx, void* stream);
/* Row passes fused into the GEMM epilogue (SURVEY §8 f1; the reference runs conv -> BatchNorm1d -> ReLU -> dropout as
 * separate full-matrix ops, arxiv_pyg/gnn.py:47-50, and autograd walks them again backwards).  Each consumer warp keeps
 * running column sums over the tiles of its CTA and stores them once: partial[slots][2][N], slots >=
 * b200gnn_gemm_stat_slots(M, N), fixed summation order (deterministic).  N a multiple of 32, 48 < N <= 256, ldc % 4 == 0.
 *   _stats_f32 : C = A·B^T + bias (accumulate: C += A·B^T, no bias — SAGEConv's lin_l(mean) + lin_r(x)) and partial = per-slot (sum C, sum C^2) over rows — the BatchNorm batch statistics of C,
 *                input of b200gnn_bn_finalize_f32 (replaces the b200gnn_col_stats_f32 sweep).
 *   _bnbwd_f32 : the input-gradient GEMM of the layer BEHIND a BatchNorm->ReLU->dropout block with pass 1 of that block's
 *                backward in the epilogue: dOut = A·B^T (+ C if accumulate); dz = dOut * [Xout > 0] / (1-p) is what is STORED
 *                to C, partial = per-slot (sum dz, sum dz*xhat), xhat = (Y-mean)*invstd (replaces
 *                b200gnn_bn_act_bwd_reduce_f32; follow with b200gnn_bn_act_bwd_apply_f32(dOut = C, Xout = NULL, sums =
 *                partial)).  Xout, Y: [M, ldc] like C. */
int64_t b200gnn_gemm_stat_slots(int64_t M, int64_t N);
/* A/B knob for measurements: 0 automatic (Xout / Y of _bnbwd_f32 staged through TMA when N % 128 == 0 and K < 128),
 * 1 = the TMA path whenever N % 128 == 0, 2 = always the register path. */
void b200gnn_gemm_set_bnbwd_variant(int v);
int b200gnn_gemm_tf32x3_stats_f32(const float* A, int64_t lda, const float* B_hi, const float* B_lo, int64_t ldb,
                                  float* C, int64_t ldc, int64_t M, int64_t N, int64_t K, const float* bias,
                                  int accumulate, float* partial, int64_t slots, void* stream);
int b200gnn_gemm_tf32x3_bnbwd_f32(const float* A, int64_t lda, const float* B_hi, const float* B_lo, int64_t ldb,
                                  float* C, int64_t ldc, int64_t M, int64_t N, int64_t K, int accumulate,
                                  const float* Xout, const float* Y, const float* mean, const float* invstd, float p_drop,
                                  float* partial, int64_t slots, void* stream);
/* Activations that are not materialised: Xout = dropout(relu(Y*scale + shift)) is recomputed from Y, the BatchNorm's
 * scale / shift and the packed keep bits of b200gnn_dropout_bits_u32 (uint32 [rows][ceil(width/32)]).
 *   _bnbwd_bits_f32 : _bnbwd_f32 with the mask [Xout > 0] taken as bit && Y*scale + shift > 0 (bits of the N columns).
 *   _act_f32        : C = Xout · B^T (+ bias) with Xout formed from Y = A in the GEMM's registers, bit for bit the
 *                     product of the materialised activation (bits of the K columns; K <= 2048). */
int b200gnn_gemm_tf32x3_bnbwd_bits_f32(const float* A, int64_t lda, const float* B_hi, const float* B_lo, int64_t ldb,
                                       float* C, int64_t ldc, int64_t M, int64_t N, int64_t K, int accumulate,
                                       const uint32_t* bits, const float* Y, const float* mean, const float* invstd,
                                       const float* scale, const float* shift, float p_drop, float* partial,
                                       int64_t slots, void* stream);
int b200gnn_gemm_tf32x3_act_f32(const float* Y, int64_t lda, const float* B_hi, const float* B_lo, int64_t ldb,
                                float* C, int64_t ldc, int64_t M, int64_t N, int64_t K, const float* bias,
                                const float* scale, const float* shift, const uint32_t* bits, float p_drop,
                                void* stream);
/* Same GEMM with the R->C layout exchange of the multi-GPU engine fused into the epilogue: output columns
 * [q*kc, (q+1)*kc), kc = N/world (a multiple of 32), are stored to C_ptrs[q][(row_off + m)*kc + ...] — C_ptrs is a HOST array
 * of `world` device pointers (the ranks' [N_nodes, kc] buffers, peer-mapped), so the tile results cross NVLink as they are
 * produced and no separate exchange kernel runs (the caller follows with b200gnn_peer_barrier). */
int b200gnn_gemm_tf32x3_scatter_f32(const float* A, int64_t lda, const float* B_hi, const float* B_lo,
                                    int64_t ldb, float* const* C_ptrs, int32_t world, int64_t row_off,
                                    int64_t M, int64_t N, int64_t K, const float* bias, void* stream);
/* ... and the row all-gather of a narrow result fused the same way: the whole [M, N] tile block is stored to EVERY
 * C_ptrs[q] (row pitch ldc) at rows row_off + m. */
int b200gnn_gemm_tf32x3_bcast_f32(const float* A, int64_t lda, const float* B_hi, const float* B_lo,
                                  int64_t ldb, float* const* C_ptrs, int32_t world, int64_t row_off, int64_t ldc,
                                  int64_t M, int64_t N, int64_t K, const float* bias, void* stream);

/* Weight gradient  dW[Kin,Nout] = X[Nn,Kin]^T * G[Nn,Nout]  (GCNConv weight.grad / nn.Linear weight.grad^T),
 * split-K over the node index on the Hopper tensor cores (wgmma, 3xTF32), partials reduced in fixed order.
 * Kin a multiple of 4 up to 2048, Nout a multiple of 4 up to 512 (else B200GNN_ERR_UNSUPPORTED); ragged edges are
 * zero-filled by TMA.  workspace: float[b200gnn_wgrad_workspace_floats(Kin,Nout)]: at most 132 node-range partials of the
 * padded [Kin, Nout] tile grid, fewer for outputs larger than 256 x 256. */
int64_t b200gnn_wgrad_workspace_floats(int64_t Kin, int64_t Nout);
int b200gnn_gemm_wgrad_tf32x3_f32(const float* X, int64_t ldx, const float* G,
                                  int64_t ldg, float* dW, int64_t Nn,
                                  int64_t Kin, int64_t Nout, float* workspace,
                                  void* stream);
/* ... with X = dropout(relu(Y*scale + shift)) recomputed from Y and the packed keep bits (uint32 [Nn][ceil(Kin/32)]). */
int b200gnn_gemm_wgrad_tf32x3_act_f32(const float* Y, int64_t ldx, const float* G, int64_t ldg, float* dW,
                                      int64_t Nn, int64_t Kin, int64_t Nout, const float* scale, const float* shift,
                                      const uint32_t* bits, float p_drop, float* workspace, void* stream);

/* ------------------------------------------------------------------ *
 * SIGN student (arxiv_dgl/sign.py:105-157): FeedForwardNet layers Linear -> PReLU (one learnable slope, a device scalar)
 * -> dropout, with the activation x = dropout(prelu(Z)) never materialised in training.  bits: packed keep decisions of
 * b200gnn_dropout_bits_u32 (bit c % 32 of word c / 32 of a row).
 *   _gemm_tf32x3_prelu_f32      : C = x · B^T (+ bias), x formed from Z in the GEMM's registers (bits uint32 [M][ceil(K/32)]),
 *                                 bit for bit the product of the activation b200gnn_prelu_bits_f32 materialises.  Any K.
 *   _gemm_tf32x3_prelu_stats_f32: _gemm_tf32x3_prelu_f32 with the BatchNorm batch statistics of C in the epilogue: output and
 *                                 partial[slots][2][N] bit for bit those of _gemm_tf32x3_stats_f32 on that activation (same
 *                                 refusals: N a multiple of 32 in (48, 256], C 16-byte aligned, ldc % 4 == 0).
 *   _gemm_tf32x3_prelu_bwd_f32  : the input-gradient GEMM behind x: dA = A · B^T (+ C if accumulate); what is STORED to C is
 *                                 dZ = (bit ? dA/(1-p) : 0) * (Z > 0 ? 1 : slope) (Z: [M, ldc] like C, bits [M][N/32], N a
 *                                 multiple of 32); slope_grad = (slope_accumulate ? slope_grad : 0) + sum over Z <= 0 of
 *                                 (bit ? dA/(1-p) : 0) * Z, reduced in fp64 per consumer warp into partial (double[slots],
 *                                 slots >= b200gnn_gemm_stat_slots(M, N)) and then in slot order: no atomics, repeatable.
 *   _gemm_wgrad_tf32x3_prelu_f32: dW = x^T · G as b200gnn_gemm_wgrad_tf32x3_f32 (Kin <= 2048), bits with a row pitch of ldbits
 *                                 words so that a wider Z runs as column blocks (Z + c0, bits + c0/32, dW + c0*Nout).
 *   _prelu_bits_f32             : out = x materialised (row pitches ldz / ldbits / ldo).
 *   _sign_gather_f32            : out[h][i] = dropout_p(feats[h][idx[i]]) for the n_hops HOST-array device pointers feats[h]
 *                                 ([n_nodes, F] each, F % 4 == 0); hop h draws the mask b200gnn_dropout_mask_u8(B, F, p, seed,
 *                                 offset + h + *step_dev * step_mul) takes.  Also labels_out[i] = labels[idx[i]] and
 *                                 teacher_out[i] = teacher[idx[i]] ([B, C], teacher pitch ldt) when given.  Indices outside
 *                                 [0, n_nodes) gather zero rows.
 *   _col_sum_ld_f32             : out[K] = column sums of Y [n_rows, K] with row pitch ldy (partial: float[slots * K], slots >=
 *                                 b200gnn_col_sum_ld_slots(n_rows)); fixed summation order.
 * ------------------------------------------------------------------ */
int b200gnn_gemm_tf32x3_prelu_f32(const float* Z, int64_t lda, const float* B_hi, const float* B_lo, int64_t ldb,
                                  float* C, int64_t ldc, int64_t M, int64_t N, int64_t K, const float* bias,
                                  const float* slope, const uint32_t* bits, float p_drop, void* stream);
int b200gnn_gemm_tf32x3_prelu_stats_f32(const float* Z, int64_t lda, const float* B_hi, const float* B_lo, int64_t ldb,
                                        float* C, int64_t ldc, int64_t M, int64_t N, int64_t K, const float* bias,
                                        const float* slope, const uint32_t* bits, float p_drop, float* partial, int64_t slots,
                                        void* stream);
int b200gnn_gemm_tf32x3_prelu_bwd_f32(const float* A, int64_t lda, const float* B_hi, const float* B_lo, int64_t ldb,
                                      float* C, int64_t ldc, int64_t M, int64_t N, int64_t K, int accumulate,
                                      const float* Z, const uint32_t* bits, const float* slope, float p_drop,
                                      float* slope_grad, int slope_accumulate, double* partial, int64_t slots,
                                      void* stream);
int b200gnn_gemm_wgrad_tf32x3_prelu_f32(const float* Z, int64_t ldz, const float* G, int64_t ldg, float* dW,
                                        int64_t Nn, int64_t Kin, int64_t Nout, const float* slope,
                                        const uint32_t* bits, int64_t ldbits, float p_drop, float* workspace,
                                        void* stream);
int b200gnn_prelu_bits_f32(const float* Z, int64_t ldz, const uint32_t* bits, int64_t ldbits, const float* slope, float p,
                           float* out, int64_t ldo, int64_t n_rows, int64_t K, void* stream);
int b200gnn_sign_gather_f32(const float* const* feats, int32_t n_hops, int64_t n_nodes, int64_t F, const int64_t* idx,
                            int64_t B, float p, uint64_t seed, uint64_t offset, const int32_t* step_dev,
                            uint64_t step_mul, float* out, const int64_t* labels, int64_t* labels_out,
                            const float* teacher, int64_t ldt, int64_t C, float* teacher_out, void* stream);
int64_t b200gnn_col_sum_ld_slots(int64_t n_rows);
int b200gnn_col_sum_ld_f32(const float* Y, int64_t ldy, int64_t n_rows, int64_t K, float* out, float* partial,
                           int64_t slots, void* stream);

/* ------------------------------------------------------------------ *
 * Feature-distillation criteria (arxiv_pyg/criterion.py): row / pair passes.
 * The S x S contractions (G-CRD logits, GSP Gram matrices) run on
 * b200gnn_gemm_tf32x3_f32; these kernels are the passes around them.
 * ------------------------------------------------------------------ */
/* F.normalize(x, p=2, dim=-1) * scale  (fitnet :30-31, gpw :68-69, nce :139-140); norm_out[n] = ||x|| */
int b200gnn_row_normalize_fwd_f32(const float* x, int64_t n, int64_t F, float eps,
                                  float scale, float* out, float* norm_out,
                                  void* stream);
int b200gnn_row_normalize_bwd_f32(const float* out, const float* norm,
                                  const float* d_out, int64_t n, int64_t F,
                                  float eps, float scale, float* d_x,
                                  int accumulate, void* stream);
/* scratch sizes for the deterministic scalar reductions below */
int64_t b200gnn_reduce_slots(int64_t n);
/* F.mse_loss(a, b): loss_out[0]; d_a (nullable) = grad_weight * 2 (a-b) / n; partial: float[b200gnn_reduce_slots(n)] */
int b200gnn_mse_fwd_bwd_f32(const float* a, const float* b, int64_t n,
                            float grad_weight, float* d_a, float* loss_out,
                            float* partial, void* stream);
/* F.binary_cross_entropy_with_logits(z, target) over n elements (ppi_pyg/criterion.py:11; target_is_logits != 0:
 * target = sigmoid(target), the teacher term of :13).  d_z (nullable) = grad_weight * (sigmoid(z) - t) / n */
int b200gnn_bce_logits_fwd_bwd_f32(const float* z, const float* target,
                                   int target_is_logits, int64_t n,
                                   float grad_weight, float* d_z, float* loss_out,
                                   float* partial, void* stream);
/* feat.pow(2).sum(-1)  (at_criterion :44-45) and its backward */
int b200gnn_row_sqnorm_f32(const float* x, int64_t n, int64_t F, float* out, void* stream);
int b200gnn_row_sqnorm_bwd_f32(const float* x, const float* d_out, int64_t n,
                               int64_t F, float* d_x, void* stream);
/* G-CRD / InfoNCE (nce_criterion :142-146) over logits Z[S,S] (already / tau):
 * loss_out[0] = mean_i(logsumexp_j Z_ij - Z_ii); Z is overwritten by d loss / d Z.  partial: float[S]. */
int b200gnn_nce_rows_f32(float* Z, int64_t S, float* loss_out, float* partial, void* stream);
/* The same pass on a ROW CHUNK of the logits (rows [row_offset, row_offset+n_rows), row pitch ldz >= S): the S x S
 * matrix of criterion.py:142-146 is never materialised — the caller streams L2-sized chunks GEMM -> this pass -> the two
 * backward GEMMs; b200gnn_nce_finish_f32 reduces partial[S] to the loss. */
int b200gnn_nce_rows_chunk_f32(float* Z, int64_t ldz, int64_t n_rows, int64_t S, int64_t row_offset,
                               float* partial, void* stream);
int b200gnn_nce_finish_f32(const float* partial, int64_t S, float* loss_out, void* stream);
/* The captured G-CRD step (csrc/gcrd.cu; nce_criterion :129-149 on the projection heads of arxiv_pyg/gnn.py:296-306).
 *   gcrd_sample: perm_out[n] = the n training-row positions ordered by (Philox key, position), keys drawn at
 *     (seed, offset + *step_dev); its first S entries are the step's sample of S distinct rows (np.random.choice(n, S,
 *     replace=False) at criterion.py:135, drawn on the device).  workspace: b200gnn_gcrd_sample_workspace_bytes(n).
 *   gcrd_operands: x_s[j] = relu(bn_s(pre_s[inds[j]])) normalised and scaled by inv_T, x_t[j] the same for the teacher
 *     head unscaled (F.normalize, eps), norms to norm_s / norm_t; pre_* [n_train, P], bn_* [4][P] (mean, invstd, scale,
 *     shift), x_* [S, P]; P a multiple of 4, at most 256.
 *   gcrd_backward: from g_* = d loss / d x_* ([S, P]) to dz_* = beta * d loss / d (bn output) at rows inds[j] of the
 *     zero-filled [n_train, P] dz_* (normalise backward, ReLU mask), and pass 1 of the BatchNorm backward: part_*[slots][2][P]
 *     (slots = b200gnn_gcrd_bwd_slots()) = per-warp (sum dz, sum dz * xhat) for b200gnn_bn_act_bwd_apply_f32 with Xout = NULL.
 *     loss_total[0] += beta * loss_aux[0] when loss_total is given. */
int64_t b200gnn_gcrd_sample_workspace_bytes(int64_t n);
int b200gnn_gcrd_sample_i32(int64_t n, uint64_t seed, uint64_t offset, const int32_t* step_dev, int32_t* perm_out,
                            void* workspace, void* stream);
int b200gnn_gcrd_operands_f32(const int32_t* inds, int64_t S, int64_t P, const float* pre_s, const float* bn_s,
                              const float* pre_t, const float* bn_t, float inv_T, float eps, float* x_s, float* x_t,
                              float* norm_s, float* norm_t, void* stream);
int64_t b200gnn_gcrd_bwd_slots(void);
int b200gnn_gcrd_backward_f32(const int32_t* inds, int64_t S, int64_t P, const float* g_s, const float* g_t,
                              const float* x_s, const float* x_t, const float* norm_s, const float* norm_t, float inv_T,
                              float eps, const float* pre_s, const float* bn_s, const float* pre_t, const float* bn_t,
                              float beta, float* dz_s, float* dz_t, float* part_s, float* part_t, const float* loss_aux,
                              float* loss_total, void* stream);
int b200gnn_transpose_f32(const float* in, int64_t rows, int64_t cols, float* out, void* stream);
/* GSP (gpw_criterion :66-86): Gs/Gt = Gram matrices of the sampled student/teacher rows; kernel 0 cosine,
 * 1 poly, 2 l2, 3 rbf (ns/nt = row squared norms for 2,3).  loss_out[0] = mse(sim_s, sim_t); Gs is overwritten by
 * d loss / d Gs; rowcoef[S] (kernels 2,3) = sum_j d loss / d ns_i.  partial: float[S]. */
int b200gnn_gsp_pair_f32(float* Gs, const float* Gt, const float* ns, const float* nt,
                         int64_t S, int kernel, float* rowcoef, float* loss_out,
                         float* partial, void* stream);
/* The chunked GSP pass: Gs / Gt = rows [row_offset, row_offset + n_rows) of the two S x S Gram matrices at row pitch
 * ld >= S, overwritten in one pass by d loss / d Gs and d loss / d Gt (each equal to what b200gnn_gsp_pair_f32 stores for
 * its side: (Gs, Gt, ns, nt) for the student, (Gt, Gs, nt, ns) for the teacher), columns S..ld-1 set to zero.  The l2 / rbf
 * diagonal and ns / nt are taken at the global row; partial[S] and (kernels 2,3) rc_s[S] / rc_t[S] are stored there, so
 * b200gnn_gsp_finish_f32 (loss_out[0] = sum partial / S^2) gives the same loss for any chunking. */
int b200gnn_gsp_pair_chunk_f32(float* Gs, float* Gt, int64_t ld, int64_t n_rows, int64_t S, int64_t row_offset,
                               const float* ns, const float* nt, int kernel, float* rc_s, float* rc_t, float* partial,
                               void* stream);
int b200gnn_gsp_finish_f32(const float* partial, int64_t S, float* loss_out, void* stream);
/* The student side of b200gnn_gsp_pair_chunk_f32 alone (a frozen teacher: Gt is read, never written; no rc_t): Gs,
 * partial and (kernels 2,3) rc_s hold the bits the two-sided pass stores for them. */
int b200gnn_gsp_pair_student_chunk_f32(float* Gs, const float* Gt, int64_t ld, int64_t n_rows, int64_t S, int64_t row_offset,
                                       const float* ns, const float* nt, int kernel, float* rc_s, float* partial,
                                       void* stream);
/* The narrow GSP contraction (csrc/loss_pair.cu): g[i, :F] (pitch ldo) = sum_{j<S} dG[i, j] x[j, :F] for the n_rows rows of
 * dG (pitch ldg >= S; columns S.. are not read) and x [S, F] (pitch ldx), in fp32 FMA.  F is a multiple of 4 up to
 * B200GNN_GSP_CONTRACT_MAX_F.  The columns are summed in slabs of B200GNN_GSP_CONTRACT_SLAB at absolute column indices,
 * ascending within a slab, and the slabs' partials are added in ascending order, so g[i] depends only on row i of dG and
 * on x (not on n_rows, the chunk a row sits in, or the device).  workspace: at least
 * b200gnn_gsp_contract_workspace_bytes(n_rows, S, F) bytes (0 when S fits one slab: workspace may be null). */
#define B200GNN_GSP_CONTRACT_MAX_F 128
#define B200GNN_GSP_CONTRACT_SLAB 256
size_t b200gnn_gsp_contract_workspace_bytes(int64_t n_rows, int64_t S, int64_t F);
int b200gnn_gsp_contract_narrow_f32(const float* dG, int64_t ldg, int64_t n_rows, int64_t S, const float* x, int64_t ldx,
                                    int64_t F, float* g, int64_t ldo, void* workspace, size_t workspace_bytes, void* stream);
/* The captured GSP step (csrc/gcrd.cu; gpw_criterion :57-92 on the projection heads of the G-CRD step).
 *   gsp_operands: kernel 0 cosine / 1 poly: x_*[j] = relu(bn_*(pre_*[inds[j]])) normalised (F.normalize, eps), its norm to
 *     norm_*[j]; kernel 2 l2 / 3 rbf: x_*[j] = relu(bn_*(pre_*[inds[j]])) and its squared norm to norm_*[j].
 *   gsp_backward: g_* = dG_* . x_* ([S, P], the chunk loop's product); the operand gradient is 2 g (kernels 0,1, then the
 *     normalise backward; norm_* required) or 2 g + 4 rc_*[j] x (kernels 2,3; rc_* required), then the ReLU mask, beta, dz_* and
 *     part_* as b200gnn_gcrd_backward_f32 stores them; loss_total[0] += beta * loss_aux[0] when loss_total is given. */
int b200gnn_gsp_operands_f32(const int32_t* inds, int64_t S, int64_t P, int kernel, const float* pre_s, const float* bn_s,
                             const float* pre_t, const float* bn_t, float eps, float* x_s, float* x_t, float* norm_s,
                             float* norm_t, void* stream);
int b200gnn_gsp_backward_f32(const int32_t* inds, int64_t S, int64_t P, int kernel, const float* g_s, const float* g_t,
                             const float* x_s, const float* x_t, const float* norm_s, const float* norm_t, const float* rc_s,
                             const float* rc_t, float eps, const float* pre_s, const float* bn_s, const float* pre_t,
                             const float* bn_t, float beta, float* dz_s, float* dz_t, float* part_s, float* part_t,
                             const float* loss_aux, float* loss_total, void* stream);
/* GSP against a fixed teacher (csrc/loss_pair.cu; the PPI step, gpw_criterion on model.out_feat and the frozen teacher's
 * out_feat, ppi_pyg/gnn.py:230-239): the teacher's n x n similarity matrix is built once, the step runs the student side.
 *   gsp_sim_chunk: sim = rows [row_offset, row_offset + n_rows) of the similarity matrix from the same rows of the Gram
 *     matrix (G pitch ldg >= n, sim pitch ld_sim >= n, both at the chunk's first row); kernels 2,3 need sq[n], the squared
 *     row norms; the l2 / rbf diagonal is exactly 0.  Each entry equals the teacher similarity b200gnn_gsp_pair_chunk_f32
 *     forms from the same Gram entry.
 *   gsp_pair_fixed_chunk: the student side of b200gnn_gsp_pair_chunk_f32 (Gs, ld, rows, ns, rc_s, partial: the same
 *     meaning and bits) with sim_t read from the stored [n_t, n_t] matrix (pitch ld_t) at [inds[i]][inds[j]]; inds[S]
 *     nullable (the identity, S <= n_t); the l2 / rbf diagonal is the sample position.
 *   gsp_rows_operands: x[j] (pitch ldx) = feat[inds[j]] (pitch ldf; inds nullable: row j) normalised with eps, norm[j] its
 *     norm (kernels 0,1: row_normalize_fwd's arithmetic), or copied, norm[j] its squared norm (kernels 2,3: row_sqnorm's).
 *   gsp_rows_backward: d_feat[inds[j]] (pitch ldd) = beta * d, d = normalise backward of 2 g[j] (kernels 0,1; norm
 *     required) or 2 g[j] + 4 rc[j] x[j] (kernels 2,3; rc required), g = dG . x; the arithmetic of row_normalize_bwd /
 *     row_axpy, then the multiply by beta.  loss_total[0] += beta * loss_aux[0] (two roundings) when loss_total is given.
 * F (the feature width) is at most B200GNN_GSP_ROWS_MAX_F, the widest layer the PPI engine stores. */
#define B200GNN_GSP_ROWS_MAX_F 2048
int b200gnn_gsp_sim_chunk_f32(const float* G, int64_t ldg, int64_t n_rows, int64_t n, int64_t row_offset, const float* sq,
                              int kernel, float* sim, int64_t ld_sim, void* stream);
int b200gnn_gsp_pair_fixed_chunk_f32(float* Gs, int64_t ld, int64_t n_rows, int64_t S, int64_t row_offset, const float* ns,
                                     const float* sim_t, int64_t ld_t, int64_t n_t, const int32_t* inds, int kernel,
                                     float* rc_s, float* partial, void* stream);
int b200gnn_gsp_rows_operands_f32(const float* feat, int64_t ldf, const int32_t* inds, int64_t S, int64_t F, int kernel,
                                  float eps, float* x, int64_t ldx, float* norm, void* stream);
int b200gnn_gsp_rows_backward_f32(const int32_t* inds, int64_t S, int64_t F, int kernel, const float* g, const float* x,
                                  int64_t ldx, const float* norm, const float* rc, float eps, float beta, float* d_feat,
                                  int64_t ldd, const float* loss_aux, float* loss_total, void* stream);
/* y[i,:] += alpha * coef[i] * x[i,:] */
int b200gnn_row_axpy_f32(const float* x, const float* coef, int64_t n, int64_t F,
                         float alpha, float* y, void* stream);

/* ------------------------------------------------------------------ *
 * LSP (lpw_criterion, arxiv_pyg/criterion.py:95-126) on an edge list sorted by
 * destination (src/dst int32[E], rowptr int32[n_seg+1] over dst).
 * kernel: 0 cosine, 1 poly, 2 l2, 3 rbf.  criterion: 0 kld, 1 mse.
 *   edge_sim     : sim[e] = k(feat[src[e]], feat[dst[e]])
 *   lsp_segment  : PyG softmax per dst segment for student and teacher sims,
 *                  loss_out[0] = the reference's loss_lpw, g[e] = d loss / d sim_s[e]
 *   edge_sim_bwd : dfeat += chain rule of g through k (atomic row adds; dfeat pre-zeroed by the caller)
 * ------------------------------------------------------------------ */
int b200gnn_edge_sim_f32(const float* feat, int64_t F, const int32_t* src,
                         const int32_t* dst, int64_t E, int kernel, float* sim,
                         void* stream);
int64_t b200gnn_lsp_partials(int64_t n_seg);
int b200gnn_lsp_segment_f32(const float* sim_s, const float* sim_t,
                            const int32_t* rowptr, int64_t n_seg, int64_t E,
                            int criterion, float* g, float* loss_out,
                            float* partial, void* stream);
int b200gnn_edge_sim_bwd_f32(const float* feat, int64_t F, const int32_t* src,
                             const int32_t* dst, int64_t E, int kernel,
                             const float* sim, const float* g, float* dfeat,
                             void* stream);
/* Deterministic LSP backward: d feat = C · feat with the (2E + n_nodes)-entry matrix C whose CSR structure
 * (comb_rowptr, and per edge / per node the entry positions pos_dst, pos_src, diag_pos) the caller builds once per
 * edge list: entry pos_dst[e] sits in row dst[e] at column src[e], pos_src[e] in row src[e] at column dst[e],
 * diag_pos[i] at (i, i).  This call fills val[2E + n_nodes] (selfc is scratch of the same size); the product itself
 * is b200gnn_spmm_csr_f32 — fixed summation order, no atomics (criterion.py:95-126 backward). */
int b200gnn_lsp_bwd_values_f32(const float* feat, int64_t F, const int32_t* src, const int32_t* dst,
                               int64_t E, int kernel, const float* sim, const float* g,
                               const int32_t* pos_dst, const int32_t* pos_src,
                               const int32_t* comb_rowptr, const int32_t* diag_pos, int64_t n_nodes,
                               float* val, float* selfc, void* stream);
/* The captured LSP step (csrc/loss_edge.cu; --training lpw, lpw_criterion :95-126 with criterion kld, on the train-induced
 * edge list of gnn_kd_and_aux.py:240-243).  The teacher similarities sim_t[E] are a constant of the run: the caller forms
 * them once with b200gnn_edge_sim_f32.
 *   lsp_student: one launch sequence for the student side, bit-identical to b200gnn_edge_sim_f32(feat) ->
 *     b200gnn_lsp_segment_f32(criterion 0) -> b200gnn_lsp_bwd_values_f32 on the same inputs: sim_s[E], val[2E + n_nodes]
 *     (diagonal included; selfc is scratch of that size) and loss_out[0].  One warp per destination segment, the segment's
 *     destination row held in registers: F (the student's width) at most B200GNN_LSP_MAX_F.  rowptr[n_seg + 1] groups the
 *     dst-sorted edges by destination, pos_* / comb_rowptr / diag_pos are the backward matrix of lsp_bwd_values;
 *     scratch: 2E floats; partial: b200gnn_lsp_partials(n_seg) floats.  Null pointers, E <= 0, n_seg <= 0, n_nodes <= 0,
 *     kernel outside 0..3 and F outside (0, B200GNN_LSP_MAX_F] are refused before any launch.
 *   scatter_rows_scaled: dst[idx[i]][k] = src[i][k] * scale (fp32 product, no FMA) for the n rows of src [n, K] (idx int64,
 *     dst row pitch ldd); no other row of dst is touched.  With loss_total, thread 0 of the launch also forms
 *     loss_total[0] = loss_total[0] + loss_aux[0] * scale (fp32 product, then fp32 add): with scale = beta this is the
 *     d (beta * loss) / d out_feat rows and the beta * loss_aux term of the step's loss, as the eager path rounds them. */
#define B200GNN_LSP_MAX_F 512
int b200gnn_lsp_student_f32(const float* feat, int64_t F, const int32_t* src, const int32_t* dst, const int32_t* rowptr,
                            int64_t n_seg, int64_t E, const float* sim_t, int kernel, const int32_t* pos_dst,
                            const int32_t* pos_src, const int32_t* comb_rowptr, const int32_t* diag_pos, int64_t n_nodes,
                            float* sim_s, float* scratch, float* val, float* selfc, float* loss_out, float* partial,
                            void* stream);
int b200gnn_scatter_rows_scaled_f32(const float* src, const int64_t* idx, int64_t n, int64_t K, float scale, float* dst,
                                    int64_t ldd, const float* loss_aux, float* loss_total, void* stream);

/* ------------------------------------------------------------------ *
 * Graph attention (BASELINE config 4): per-destination edge softmax and
 * multi-head weighted aggregation, CSR rows = destinations, col = sources.
 *   DGL GATConv.forward   arxiv_dgl/models.py:196-217  (softmax_eps = 0)
 *   PyG GATConv           ppi_pyg/gnn.py:27-31          (softmax_eps = 1e-16)
 *   gat_edge_softmax : a[e,h] = softmax_e( leaky_relu(el[col[e],h] + er[row,h]) )   er NULL => el only
 *   gat_aggregate    : out[r, h*D+d] = sum_e a[eidx ? eidx[e] : e, h] * ft[col[e], h*D+d]
 *                      (forward on the CSR; d ft on the transposed CSR with eidx = csr2csc)
 *   gat_bwd_rows     : given d out, writes dpre[e,h] = d loss / d (el+er)[e,h] and der[r,h]
 *   segment_sum_heads: out[r,h] = sum_e vals[eidx[e],h]  (d el over the transposed CSR)
 * H <= 16.  chunk_rowptr / hub_rows / hub_segptr: the plans of b200gnn_csr_chunk_plan / b200gnn_csr_hub_fill
 * (rows above hub_threshold are split into seg_len-edge segments, as in b200gnn_spmm_csr_f32).
 * hub_workspace: n_seg*H*D floats for gat_aggregate, n_seg*H floats for gat_bwd_rows (unused when n_hub == 0).
 * Teacher-training knobs (arxiv_dgl/models.py:206-214): edge_keep [nnz] uint8 (NULL = keep all) — dropped edges get
 * a = 0 and leave the softmax (edge_drop); attn_scale [nnz,H] (NULL = none) = keep/(1-p) of the attention dropout:
 * the caller aggregates with a*attn_scale and gat_bwd_rows chains d a = d(a*attn_scale) * attn_scale.
 * ------------------------------------------------------------------ */
int b200gnn_gat_edge_softmax_f32(const int32_t* rowptr, const int32_t* col,
                                 const float* el, const float* er, int64_t n_rows,
                                 int64_t H, float negative_slope, float softmax_eps,
                                 float* a, const uint8_t* edge_keep, void* stream);
int b200gnn_gat_aggregate_f32(const int32_t* rowptr, const int32_t* col,
                              const int32_t* eidx, const float* a, const float* ft,
                              int64_t ldf, float* out, int64_t ldo, int64_t n_rows,
                              int64_t H, int64_t D, const int32_t* chunk_rowptr,
                              int64_t n_chunks, int32_t hub_threshold, int32_t seg_len,
                              const int32_t* hub_rows, const int32_t* hub_segptr,
                              int64_t n_hub, int64_t n_seg, float* hub_workspace,
                              void* stream);
int b200gnn_gat_bwd_rows_f32(const int32_t* rowptr, const int32_t* col, const float* a,
                             const float* ft, int64_t ldf, const float* dout,
                             int64_t ldd, const float* el, const float* er,
                             int64_t n_rows, int64_t H, int64_t D,
                             float negative_slope, float* dpre, float* der,
                             const int32_t* chunk_rowptr, int64_t n_chunks,
                             int32_t hub_threshold, int32_t seg_len,
                             const int32_t* hub_rows, const int32_t* hub_segptr,
                             int64_t n_hub, int64_t n_seg, float* hub_workspace,
                             const float* attn_scale, void* stream);
int b200gnn_segment_sum_heads_f32(const int32_t* rowptr, const int32_t* eidx,
                                  const float* vals, int64_t n_rows, int64_t H,
                                  float* out, void* stream);

/* ------------------------------------------------------------------ *
 * The fused GAT layer of the full-batch trainer (engine_gat.py): what the reference's GATConv.forward runs as separate
 * [N, H*D] torch ops around its two DGL kernels.
 *   gat_scores        : el[n,h] = src_scale[n] * <ft[n,h,:], attn_l[h,:]>, er[n,h] = <ft[n,h,:], attn_r[h,:]> in one read of
 *                       ft (row pitch ldf) — arxiv_dgl/models.py:179-184 (feat_src * out_deg^-1/2), :196 (el), :200 (er from
 *                       the un-normalised projection).  src_scale / attn_r (with er) may be NULL.  One warp per node, fixed
 *                       summation order.
 *   gat_scores_bwd    : dft[n,h,:] += d_el[n,h] src_scale[n] attn_l[h,:] + d_er[n,h] attn_r[h,:] in place, d_attn_l[h,:] =
 *                       sum_n d_el[n,h] src_scale[n] ft[n,h,:], d_attn_r[h,:] = sum_n d_er[n,h] ft[n,h,:] (autograd of
 *                       models.py:196,200): per-CTA partials over contiguous row blocks (partial: [slots][2][H*D] floats,
 *                       slots >= b200gnn_gat_scores_slots(n_rows)) added in slot order — no atomics, repeatable.  H*D <= 1536.
 *   gat_aggregate_epi : b200gnn_gat_aggregate_f32 (same plans, same summation order) with the rest of the layer in its
 *                       epilogue: out[i,:] = row_scale[i] * sum_e a[e,h] src_scale[col[e]] ft[col[e],h,:] + res[i,:] + bias
 *                       (models.py:184 folded into the coefficient, :220-225 in_deg^+1/2, :228-230 residual, :311
 *                       bias_last), and stat_partial[slots][2][H*D] = per-CTA (sum, sum of squares) of the output rows,
 *                       slots >= b200gnn_gat_stat_slots(n_chunks, n_hub), the input of b200gnn_bn_finalize_f32
 *                       (models.py:304's BatchNorm1d statistics).  Every epilogue operand may be NULL; with all of them
 *                       NULL the output equals b200gnn_gat_aggregate_f32's bit for bit.  Run on the transposed graph with
 *                       the two scale vectors exchanged it is the backward aggregation (d ft).
 * ------------------------------------------------------------------ */
int b200gnn_gat_scores_f32(const float* ft, int64_t ldf, const float* attn_l, const float* attn_r,
                           const float* src_scale, int64_t n_rows, int64_t H, int64_t D, float* el, float* er,
                           void* stream);
int64_t b200gnn_gat_scores_slots(int64_t n_rows);
int b200gnn_gat_scores_bwd_f32(const float* ft, int64_t ldf, const float* attn_l, const float* attn_r,
                               const float* src_scale, const float* d_el, const float* d_er, int64_t n_rows,
                               int64_t H, int64_t D, float* dft, int64_t ldd, float* d_attn_l, float* d_attn_r,
                               float* partial, int64_t slots, void* stream);
int64_t b200gnn_gat_stat_slots(int64_t n_chunks, int64_t n_hub);
int b200gnn_gat_aggregate_epi_f32(const int32_t* rowptr, const int32_t* col, const int32_t* eidx, const float* a,
                                  const float* ft, int64_t ldf, float* out, int64_t ldo, int64_t n_rows, int64_t H,
                                  int64_t D, const float* src_scale, const float* row_scale, const float* res,
                                  int64_t ldr, const float* bias, float* stat_partial, int64_t stat_slots,
                                  const int32_t* chunk_rowptr, int64_t n_chunks, int32_t hub_threshold,
                                  int32_t seg_len, const int32_t* hub_rows, const int32_t* hub_segptr, int64_t n_hub,
                                  int64_t n_seg, float* hub_workspace, void* stream);

/* ------------------------------------------------------------------ *
 * The PyG GAT layers of the PPI models (engine_ppi.py; ppi_pyg/gnn.py:24-83): hidden layers x = elu(GATConv(x) + Linear(x)),
 * a last layer GATConv(concat=False) + Linear.
 *   gat_aggregate_elu : b200gnn_gat_aggregate_epi_f32 with res / bias (no scale vectors, no statistics) that also stores
 *                       act = elu(out) (row pitch lda): out = Z is the epi entry point's output bit for bit (same plans,
 *                       same vector width and summation order, hub rows through the same finalize), act is the next layer's
 *                       GEMM operand.  act must admit the vector width the epi entry point picks for the other operands
 *                       (16-byte base and lda % 4 == 0 when out / ft / res / bias do; 8-byte and even lda for the float2
 *                       path), else B200GNN_ERR_BAD_ARG.
 *   elu_bwd           : dZ = dA * (Z > 0 ? 1 : exp(Z)) (torch's elu_backward), every operand with its own row pitch.
 *   ppi_logits_loss   : logits[r, c] = (mean_h agg[r, h*Dp + c] + b_conv[c]) + (res[r, c] + b_lin[c]) for c < C (agg [n, H*Dp]
 *                       from the plain aggregation, res [n, >= Dp]).  With labels (float multi-hot, [n, C] pitch ldy) also
 *                       the loss over all n*C entries: BCE-with-logits, or with teacher logits the logit KD alpha T^2
 *                       BCE(z, sigmoid(t)) + (1 - alpha) BCE(z, y); loss_out[3] = [loss, loss_cls, loss_kd] ([cls, cls, 0]
 *                       without a teacher); d_agg[r, h*Dp + c] = dz / H in every head, d_res[r, c] = dz, columns C..Dp-1
 *                       of both written as zero.  Per-CTA fp64 sums in partial (double[2 * slots], slots >=
 *                       b200gnn_ppi_tail_slots(n)), added in slot order: no atomics, repeatable.  Without labels only the
 *                       logits are written (eval).
 * ------------------------------------------------------------------ */
int b200gnn_gat_aggregate_elu_f32(const int32_t* rowptr, const int32_t* col, const int32_t* eidx, const float* a,
                                  const float* ft, int64_t ldf, float* out, int64_t ldo, float* act, int64_t lda,
                                  int64_t n_rows, int64_t H, int64_t D, const float* res, int64_t ldr,
                                  const float* bias, const int32_t* chunk_rowptr, int64_t n_chunks,
                                  int32_t hub_threshold, int32_t seg_len, const int32_t* hub_rows,
                                  const int32_t* hub_segptr, int64_t n_hub, int64_t n_seg, float* hub_workspace,
                                  void* stream);
int b200gnn_elu_bwd_f32(const float* dA, int64_t ldda, const float* Z, int64_t ldz, float* dZ, int64_t lddz,
                        int64_t n_rows, int64_t K, void* stream);
int64_t b200gnn_ppi_tail_slots(int64_t n_rows);
int b200gnn_ppi_logits_loss_f32(const float* agg, int64_t lda, const float* res, int64_t ldr, const float* b_conv,
                                const float* b_lin, int64_t n_rows, int64_t H, int64_t Dp, int64_t C,
                                float* logits, int64_t ldl, const float* labels, int64_t ldy,
                                const float* teacher_logits, int64_t ldt, float alpha, float T, float* d_agg,
                                int64_t ldga, float* d_res, int64_t ldgr, float* loss_out, double* partial,
                                int64_t slots, void* stream);

/* ------------------------------------------------------------------
 * Peer-memory exchange of the node-parallel engine (SURVEY.md §8e; no reference counterpart: the reference is
 * single-GPU, arxiv_pyg/scripts/run_gcn.sh:24-28).  One process per GPU; each rank allocates an exchange arena,
 * publishes its CUDA IPC handle (64 opaque bytes, exchanged by the host side, e.g. torch.distributed) and maps the
 * peers' arenas.  Exchange steps are kernels that store directly into the consumers' arenas over NVLink, then a
 * flag barrier:
 *   b200gnn_peer_copy2d_f32 : n <= 16 strided block copies in one launch, dst_j[r, 0:width] = src_j[r, 0:width]
 *                             (width % 4 == 0; 16-byte aligned bases and pitches); dst_j may be peer memory
 *   b200gnn_peer_barrier    : peer_flags[q] = rank q's flag array (16 uint64 slots, zero-initialised, inside its
 *                             arena) as mapped in THIS process (host array of `world` device pointers); stores
 *                             epoch+1 into slot [rank] of every rank's array with release semantics at system
 *                             scope, waits until its own slots all reached it, then bumps *epoch (device counter,
 *                             so the call is CUDA-graph replayable).  A peer that never arrives sets *error = 1
 *                             after ~2^27 polls instead of hanging the device.
 * ------------------------------------------------------------------ */
typedef struct b200gnn_copy2d {
  float* dst;
  const float* src;
  int64_t ld_dst; /* floats */
  int64_t ld_src; /* floats */
  int64_t rows;
} b200gnn_copy2d;
int b200gnn_arena_alloc(int64_t bytes, void** out);
int b200gnn_arena_free(void* ptr);
int b200gnn_ipc_get_handle(const void* dev_ptr, void* handle64);
int b200gnn_ipc_open_handle(const void* handle64, void** out);
int b200gnn_ipc_close_handle(void* ptr);
int b200gnn_peer_copy2d_f32(const b200gnn_copy2d* copies, int32_t n, int64_t width, void* stream);
int b200gnn_peer_barrier(uint64_t* const* peer_flags, int32_t rank, int32_t world,
                         uint64_t* epoch, int32_t* error, void* stream);
/* copy2d + barrier in ONE launch: the CTA that finishes last (ticket: device uint32, zero-initialised, re-armed by the
 * kernel) runs the flag barrier, so the kernel ends when every rank's blocks have been exchanged. */
int b200gnn_peer_exchange_f32(const b200gnn_copy2d* copies, int32_t n, int64_t width,
                              uint64_t* const* peer_flags, int32_t rank, int32_t world, uint64_t* epoch,
                              int32_t* error, uint32_t* ticket, void* stream);

/* ------------------------------------------------------------------
 * Heterogeneous input assembly — RGCN.group_input, mag_pyg/gnn.py:111-124 (called from RGCN.forward :126-129):
 *   out[i, :] = tables[node_type[i]][local_idx[i], :]     (tables[t] NULL or type out of range => zero row)
 * node_type / local_idx are the int64 tensors of group_hetero_graph; tables / table_rows are HOST arrays of
 * n_tables <= 16 device pointers / row counts.  An index outside its table sets *error_flag (device int32) to 1.
 * typed_scatter is the backward: d_tables[t][j, :] = sum over nodes i with (node_type, local_idx) == (t, j) of
 * d_out[i, :], written (not accumulated: untouched rows keep what the caller put there, normally zeros) for the
 * tables whose pointer is non-NULL.  `order` = the node ids sorted by (node_type, local_idx) (stable): runs of equal
 * keys are added in that order by one warp => deterministic, no atomics.
 * ------------------------------------------------------------------ */
int b200gnn_typed_gather_f32(const float* const* tables, const int64_t* table_rows, int32_t n_tables,
                             const int64_t* node_type, const int64_t* local_idx, int64_t n, int64_t F,
                             float* out, int64_t ldo, int32_t* error_flag, void* stream);
/* Adam over ONE embedding table (rows x F; the table of node type table_type) whose gradient is the typed_scatter of
 * d_out: row j's gradient is the sum of the d_out rows of the nodes with (node_type, local_idx) == (table_type, j), added in
 * `order`, or 0 if there is none, and every row of the table gets the b200gnn_adam_step_f32 update.  Bit-identical to
 * b200gnn_typed_scatter_f32 into a zeroed table followed by b200gnn_adam_step_f32, without the dense gradient.
 * order: the n nodes sorted by (node_type, local_idx).  head: int32[rows] scratch, all -1 on entry, restored on return.
 * *step is read (steps already taken) and NOT incremented: the flat-buffer b200gnn_adam_step_f32 that runs after it
 * owns the counter. */
int b200gnn_embedding_adam_f32(const float* d_out, int64_t ldd, const int64_t* node_type,
                               const int64_t* local_idx, const int64_t* order, int64_t n,
                               int64_t table_type, float* table, float* exp_avg, float* exp_avg_sq,
                               int64_t rows, int64_t F, int32_t* head, float lr, float beta1,
                               float beta2, float eps, const int32_t* step, void* stream);
int b200gnn_typed_scatter_f32(const float* d_out, int64_t ldd, const int64_t* node_type,
                              const int64_t* local_idx, const int64_t* order, int64_t n, int64_t F,
                              float* const* d_tables, const int64_t* table_rows, int32_t n_tables,
                              void* stream);

/* ------------------------------------------------------------------
 * Graph ingestion on the device (SURVEY.md §8 f2) — the integer half of the data path, bit-exact:
 *   b200gnn_graph_argsort_i64  : perm = stable argsort of key = major*minor_size + minor.  ToSparseTensor
 *                                (arxiv_pyg/gnn.py:236-237: major = edge_index[1], minor = edge_index[0]), an unsorted
 *                                SparseTensor(row=, col=) (mag_pyg/gnn.py:151) and csr2csc (major = col, minor = row).
 *   b200gnn_graph_coalesce_i64 : COO -> row-sorted duplicate-free COO + rowptr (to_symmetric's coalesce,
 *                                arxiv_pyg/gnn.py:240).  out_row/out_col/src_out hold n entries, the first *nnz_out
 *                                (device int64) are valid; src_out (nullable) = input index of each kept entry.
 * Hand-written stable LSD radix sort (8-bit digits, only the digits the key range needs) + flags/scan/compaction +
 * binary-search row pointers.  workspace: b200gnn_graph_sort_workspace_bytes(n) bytes, 256-byte aligned.
 * n < 2^31; major_size*minor_size < 2^64.
 * ------------------------------------------------------------------ */
int64_t b200gnn_graph_sort_workspace_bytes(int64_t n);
int b200gnn_graph_argsort_i64(const int64_t* major, const int64_t* minor, int64_t n, int64_t major_size,
                              int64_t minor_size, int32_t* perm_out, void* workspace, void* stream);
int b200gnn_graph_coalesce_i64(const int64_t* row, const int64_t* col, int64_t n, int64_t n_rows,
                               int64_t n_cols, int64_t* out_row, int64_t* out_col, int32_t* src_out,
                               int64_t* rowptr_out, int64_t* nnz_out, void* workspace, void* stream);

/* ------------------------------------------------------------------
 * Mini-batch sampling on the device (SURVEY §8 f4) — replaces the CPU workers of
 * torch_geometric.data.GraphSAINTRandomWalkSampler as the reference drives it (mag_pyg/gnn.py:361-366: roots uniform
 * over the nodes, torch_sparse.random_walk of walk_length steps, SparseTensor.saint_subgraph of the visited nodes).
 *   random_walk: out[w][0] = start[w]; step s of walker w moves to col[rowptr[v] + (r * deg >> 32)], r = word (s % 4) of
 *     Philox4x32-10(seed, offset, w * ceil(L/4) + s / 4); a node without out-edges holds the walker.  out: [n_walks, L+1].
 *   saint_subgraph: induced subgraph of the sorted unique node set `nodes` over CSR, CSR order kept.  count -> per selected
 *     row the number of kept edges (and fills node_map, an int32 [n_nodes] workspace that holds -1 on entry); the caller
 *     prefix-sums the counts into out_ptr; fill -> local row / local col / parent edge id (eid[j], or j when eid is NULL).
 *   induced_edges: the edges of edge_index (int64 rows: src at edge_index[0..E), dst at edge_index[ld..ld+E)) whose two
 *     endpoints are marked in mask (uint8 / bool [n_nodes]), relabelled to the endpoints' ranks among the marked nodes, edge
 *     order kept: torch_geometric.utils.subgraph(mask.nonzero(), edge_index, relabel_nodes=True)[0].  count -> rank (int64
 *     [n_nodes + 1] workspace: marked nodes before each node, rank[n_nodes] = all of them), tile_cnt (int64
 *     [2 * b200gnn_induced_edges_tiles(E)] workspace) and totals (int64 [2]: kept edges, edges with an endpoint outside
 *     [0, n_nodes), which are never kept); fill -> out[0..kept) sources and out[ld_out..ld_out + kept) destinations, reading
 *     the rank and tile_cnt the count call left.
 * ------------------------------------------------------------------ */
int b200gnn_random_walk_i64(const int32_t* rowptr, const int32_t* col, int64_t n_nodes, const int64_t* start,
                            int64_t n_walks, int32_t walk_length, uint64_t seed, uint64_t offset, int64_t* out,
                            void* stream);
int b200gnn_saint_subgraph_count_i64(const int32_t* rowptr, const int32_t* col, const int64_t* nodes, int64_t n_sel,
                                     int32_t* node_map, int64_t* counts, void* stream);
int b200gnn_saint_subgraph_fill_i64(const int32_t* rowptr, const int32_t* col, const int64_t* eid, const int64_t* nodes,
                                    int64_t n_sel, const int32_t* node_map, const int64_t* out_ptr, int64_t* out_row,
                                    int64_t* out_col, int64_t* out_eid, void* stream);
int64_t b200gnn_induced_edges_tiles(int64_t n_edges);
int b200gnn_induced_edges_count_i64(const int64_t* edge_index, int64_t ld, int64_t n_edges, const uint8_t* mask,
                                    int64_t n_nodes, int64_t* rank, int64_t* tile_cnt, int64_t* totals, void* stream);
int b200gnn_induced_edges_fill_i64(const int64_t* edge_index, int64_t ld, int64_t n_edges, const uint8_t* mask,
                                   int64_t n_nodes, const int64_t* rank, const int64_t* tile_cnt, int64_t* out,
                                   int64_t ld_out, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* B200GNN_H_ */
