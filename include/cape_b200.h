/*
 * cape_b200.h -- C ABI of libcape_b200.so: the H100 (sm_90a) implementation of CAPE's graph-conv hot path.
 *
 * The reference (qianlim/CAPE, TF-1.13) has no FFI; its operator seam is name-based dispatch on
 * `base_model` (lib/models.py:16-17,58-62: filter='chebyshev5', pool/unpool='poolwT',
 * activation='b1leakyrelu').  Each entry point below cites the reference op(s) it replaces.  A maintainer
 * of the reference would bind these with ctypes (INTEGRATION.md shows the stub).
 *
 * Conventions
 *   - every function returns 0 on success, <0 on error; cape_last_error() gives the message (thread-local);
 *     no C++ exception crosses the boundary.
 *   - all tensors are fp32, row-major, caller-owned DEVICE pointers; feature tensors are [N, rows, F] with F
 *     contiguous (the reference's [N, M, F] placeholders, lib/models.py:272-282).
 *   - every kernel is enqueued on the caller's `stream` (a cudaStream_t passed as void*); no hidden
 *     synchronisation, no allocation inside hot calls (workspace is owned by the topology handle).
 *   - the topology handle is immutable after the last cape_topology_add_operator() and may be shared
 *     across streams of one device.
 */
#ifndef CAPE_B200_H
#define CAPE_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define CAPE_ABI_VERSION 4
#define CAPE_MAX_TERMS 8

typedef struct cape_topology cape_topology;

/* ---- error / version --------------------------------------------------------------------------- */
const char* cape_last_error(void);
int cape_abi_version(void);
/* number of CUDA kernels this library has launched in this process (bench.py reports it as gpu_launches) */
int64_t cape_launch_count(void);

/* ---- topology handle: the fixed sparse operators ------------------------------------------------
 * Replaces the graph-build-time conversion of scipy matrices into tf.SparseTensor
 * (lib/models.py:74-79 for the rescaled Laplacian, :141-145 for D/U).
 * An operator is a sparse [rows_out x rows_in] matrix in ELL form: idx/w are [rows_out, width] row-major,
 * unused slots have idx = -1.  The host composes D * T_k(L~) * U offline (cape_b200/topology.py) so that
 * pooling (lib/models.py:168) and unpooling (:750,:782) are folded into the conv's neighbour gather.
 * The library also keeps each operator's row sums (the constants c_k of the condition broadcast,
 * lib/models.py:813-832).  Returns the operator id (>=0) or <0. */
int cape_topology_create(int device, cape_topology** out);
void cape_topology_destroy(cape_topology* t);
int cape_topology_add_operator(cape_topology* t, int rows_out, int rows_in, int width,
                               const int32_t* idx_host, const float* w_host);
/* split-K / partial-sum workspace used by the dW and GEMM kernels (bytes); call once before hot calls. */
int cape_topology_reserve_workspace(cape_topology* t, int64_t bytes);

/* ---- fused Chebyshev graph convolution ----------------------------------------------------------
 * One term = one polynomial order (or one branch of a block):
 *   A_t[n, r, f] = sum_j w_op[r, j] * src[n, idx_op[r, j], f]        (op < 0: identity, A_t = src)
 *   acc0 (and acc1 if w2) += A_t[:, :, :F] @ W_t[:F, :ncols],   W_t element (f, c) = w[f * w_stride + c]
 * plus the condition broadcast without materialising it (lib/models.py:591-594,606-609,663-666):
 *   acc += rowsum(op)[r] * (cond[n, :C] @ Wc_t[:C, :ncols]),    Wc_t element (j, c) = wc[j * w_stride + c]
 * A term whose w, w2, wT and w2T are all NULL is a PASS-THROUGH term: no contraction,
 *   acc0 += A_t[:, :, :ncols]      (a residual added before the epilogue's bias / activation / SLOPE mask)
 * It needs F == ncols and takes no wc, wc2 or stash; a call needs at least one contracted term, and a plain_only call
 * takes no pass-through term (rc < 0 otherwise).
 */
typedef struct {
  const float* src;   /* [N, src_rows, src_stride] */
  int op;             /* operator id, or -1 for identity */
  int F;              /* reduction length (channels of src used) */
  int src_rows;
  int src_stride;     /* floats between consecutive rows of src (>= F) */
  int w_stride;       /* floats between consecutive reduction rows of w / wc */
  int w2_stride;      /* same for w2 / wc2 */
  const float* w;     /* -> accumulator 0 */
  const float* w2;    /* -> accumulator 1 (NULL: none) */
  const float* wc;    /* condition rows for accumulator 0 (NULL: none) */
  const float* wc2;   /* condition rows for accumulator 1 (NULL: none) */
  /* optional K-major copies of w / w2 (element (f, c) = wT[c * wT_stride + f]); when given for every term and the
   * shapes allow it the contraction runs on the wgmma tensor cores (3xTF32, fp32-accurate), else on the fp32 pipe */
  const float* wT;
  const float* w2T;
  int wT_stride;
  int w2T_stride;
  /* optional: also write this term's gathered basis rows  B[n, r, 0:F] = sum_j op[r, j] * src[n, idx[r, j], 0:F]  to
   * stash[(n * rows_out + r) * stash_stride + f]  (16-byte aligned, stash_stride % 4 == 0, F % 4 == 0).  The weight
   * gradient of the layer can then contract plain tensors (cape_cheb_dw with op = -1: the dense-operand kernel) instead of
   * gathering again: in a forward call the stash is the basis itself, in a data-gradient call it is op^T . G, the
   * "narrow side" operand (dW_k = x^T (op_k^T G)). */
  float* stash;
  int stash_stride;
} cape_term;

enum {
  CAPE_EPI_LINEAR = 0,   /* out = act(acc0 + bias)                       chebyshev5 + b1leakyrelu, models.py:69-109 */
  CAPE_EPI_AFFINE = 1,   /* out = acc1 + relu(acc0); out2 = relu(acc0)   res_block_affine, models.py:776-793 */
  CAPE_EPI_SLOPE = 2,    /* out = acc0 * (aux > 0 ? 1 : alpha)           backward through (leaky-)ReLU given its output */
  CAPE_EPI_DUALMASK = 3, /* out = acc0; out2 = acc0 * (aux > 0)          backward into an affine block's output */
  CAPE_EPI_TANHGRAD = 4  /* out = acc0 * (1 - aux^2)                     backward through tanh given its output
                          * (b1tanh, models.py:111-115); ReLU (b1relu, :117-121) is SLOPE with alpha = 0 */
};
/* LEAKY: b1leakyrelu (models.py:105-109), RELU: b1relu (:117-121), TANH: b1tanh (:111-115, the precise tanhf) */
enum { CAPE_ACT_NONE = 0, CAPE_ACT_LEAKY = 1, CAPE_ACT_RELU = 2, CAPE_ACT_TANH = 3 };

typedef struct {
  int N, rows_out, ncols;
  int nterms;
  cape_term terms[CAPE_MAX_TERMS];
  const float* cond;   /* [N, C] condition embedding (NULL: none) */
  int C;
  int epilogue;        /* CAPE_EPI_* */
  int act;             /* CAPE_ACT_* (LINEAR only) */
  float alpha;         /* negative slope (LEAKY: 0.2 = tf.nn.leaky_relu default; SLOPE epilogue) */
  const float* bias;   /* [ncols] or [rows_out, ncols] (NULL: none) */
  int bias_per_row;    /* 1: per-vertex bias (decoder outputs, models.py:615) */
  const float* aux;    /* [N, rows_out, ncols] (SLOPE / DUALMASK / TANHGRAD) */
  float* out;          /* [N, rows_out, ncols] */
  float* out2;         /* [N, rows_out, ncols] or NULL */
  /* 1: fail (rc < 0) instead of falling back to the gather / fp32-pipe kernels when the plain-operand tensor-core kernel
   * cannot take the call -- for callers that only filled wT / w2T (the `w` pointers are then never read). */
  int plain_only;
} cape_conv_args;

/* ---- operators without contraction: the gather half of the split conv forms -----------------------------
 *   acc_a[n, r, c] = sum_{t: acc_t = a} scale_t * ( sum_j op_t[r, j] * src_t[n, idx_t[r, j], c]
 *                                                   + rowsum(op_t)[r] * (cond[n, :C] @ wc_t[:C, c]) ),     c < ncols
 * then the epilogue of cape_conv_args (LINEAR: bias + activation; AFFINE: out = acc1 + relu(acc0), out2 = relu(acc0);
 * SLOPE / DUALMASK with aux).  With the tensor-core contraction of plain tensors (cape_cheb_fwd, all terms identity) this
 * gives the two split forms of chebyshev5 (+poolwT, +fit_cond_dim; lib/models.py:69-103,129-152,813-832):
 *   contract first:  Z = X @ [W_0 | W_1 | ...]   (cape_cheb_fwd),   out = epi(sum_k op_k Z_k)   (cape_apply)
 *   basis first:     B_k = op_k X                 (cape_apply),      out = epi(sum_k B_k W_k)    (cape_cheb_fwd)
 * and single steps of the Chebyshev recurrence (T_k x = 2 L~ T_{k-1} x - T_{k-2} x: two terms, scales 2 and -1). */
typedef struct {
  const float* src;   /* [N, src_rows, src_stride]; channels [0, ncols) are used */
  int op;             /* operator id ([rows_out x src_rows]), or -1 for identity */
  int src_rows;
  int src_stride;     /* floats between rows of src (>= ncols, % 4 == 0) */
  int acc;            /* accumulator 0 or 1 */
  float scale;        /* factor of the term (0 means 1) */
  const float* wc;    /* optional condition rows [C, >= ncols] for this term (NULL: none) */
  int wc_stride;      /* floats between rows of wc */
} cape_apply_term;

typedef struct {
  int N, rows_out, ncols;    /* ncols % 4 == 0, <= 1024 */
  int nterms;
  cape_apply_term terms[CAPE_MAX_TERMS];
  const float* cond;   /* [N, C] (NULL: none) */
  int C;
  int epilogue, act;   /* CAPE_EPI_*, CAPE_ACT_* */
  float alpha;
  const float* bias;   /* [ncols] or [rows_out, ncols] */
  int bias_per_row;
  const float* aux;    /* [N, rows_out, ncols] (SLOPE / DUALMASK / TANHGRAD) */
  float* out;          /* rows out_stride floats apart (0: ncols) -- the result may land inside a wider buffer */
  int out_stride;
  float* out2;         /* same stride, or NULL */
  /* > 0: "separate" mode -- no summation and no epilogue, term t is written on its own to out + t * term_stride floats
   * (the K basis tensors B_k = op_k x of a layer in ONE launch; LINEAR epilogue, no bias / activation / condition) */
  int64_t term_stride;
} cape_apply_args;
int cape_apply(cape_topology* t, const cape_apply_args* a, void* stream);

/* Experiment knobs (process-wide, all 0 by default = the shipped configuration).  They switch single
 * optimisations off for A/B measurements and fallback-path tests: [7]=1 thin-output layers on the generic kernels,
 * [8]=1 no tensor-core plain-operand conv path, [10]=rows per CTA of cape_apply (16..1024), [11]=chunks of 32 rows
 * per MMA chain of the tensor-core weight gradient (0: 64, <0: one chain per row split), [16]=1 scalar FC kernel,
 * [17]=1 fixed CTA count of the thin weight gradient.  Returns the previous value, <0 for an unknown key. */
int cape_set_tuning(int key, int value);

/* Process-wide switch for the tensor-core path of cape_cheb_fwd (default on); returns the previous setting. */
int cape_set_tensor_cores(int enable);
int cape_tensor_cores_enabled(void);

/* Forward of chebyshev5 (+poolwT, +b1leakyrelu, +fit_cond_dim/concat) -- lib/models.py:69-103,105-109,
 * 129-152,813-832; also the data-gradient pass (same form with transposed operators and weights). */
int cape_cheb_fwd(cape_topology* t, const cape_conv_args* a, void* stream);

/* Weight gradient of one term:  dw[f * dw_stride + c] (+)= sum_{n,r} A_t[n,r,f] * g[n,r,c]
 * (TF autodiff of lib/models.py:102; deterministic split-K through the topology workspace). */
typedef struct {
  int N, rows_out, ncols;
  const float* src; int op; int F; int src_rows; int src_stride;
  const float* g;      /* [N, rows_out, ncols] */
  float* dw; int dw_stride;
  int accumulate;      /* 0: overwrite, 1: add */
  /* optional: all the terms of one layer in one call (one pass over g when the input is thin): operators ops[0..nops)
   * instead of `op`, term j written to dw + j * dw_term_stride.  nops = 0: the single term `op`. */
  int nops;
  int ops[CAPE_MAX_TERMS];
  int dw_term_stride;
  /* with nops > 0 and a thin input (F <= 4): element (f, c) of term j goes to
   * dw[j * dw_term_stride + f * dw_stride + c * dw_col_stride]  (0 = 1).  Lets the caller swap the operand roles for
   * thin-OUTPUT layers -- dW_j^T = (op_j^T g)^T x, the operators applied to the 3-channel gradient -- and still get
   * dW in the [Fin, K, Fout] layout. */
  int dw_col_stride;
} cape_dw_args;
int cape_cheb_dw(cape_topology* t, const cape_dw_args* a, void* stream);

/* Per-sample weighted column sums: out[n, j, c] = sum_r rowsum(op_j)[r] * g[n, r, c]  (op_j < 0: ones); rows of g
 * are g_stride floats apart (>= ncols).  Gives the bias gradient (models.py:105-109) and the gradient of the
 * condition broadcast (the reduce-over-vertices implied by fit_cond_dim, models.py:829-830).  out is ACCUMULATED
 * into (zero it first). */
int cape_colsum(cape_topology* t, const float* g, int g_stride, int N, int rows, int ncols,
                const int* ops, int nops, float* out, void* stream);

/* ---- dense layers (tf.layers.dense, lib/models.py:496,506,510,557,560,582) ------------------------
 * C[M,N] = act(alpha * A.B + bias) (+ beta * C);  A(m,k) = a[m*a_rs + k*a_cs], B(k,n) = b[k*b_rs + n*b_cs]. */
int cape_gemm(cape_topology* t, int M, int N, int K,
              const float* a, int64_t a_rs, int64_t a_cs,
              const float* b, int64_t b_rs, int64_t b_cs,
              float* c, int64_t c_rs,
              const float* bias, int act, float leaky_alpha, float alpha, float beta, void* stream);

/* cape_gemm followed by a data-gradient epilogue of the conv kernels, applied last (after the beta accumulation):
 *   CAPE_EPI_LINEAR    C as cape_gemm writes it (aux unread);
 *   CAPE_EPI_SLOPE     C *= (aux > 0 ? 1 : epi_alpha)      (leaky ReLU / ReLU backward given the layer's output);
 *   CAPE_EPI_TANHGRAD  C *= 1 - aux^2                      (tanh backward given the layer's output);
 * aux(m, n) = aux[m*aux_rs + n], C's shape.  The FC layers' input gradient at reduce_dim 0 is this product: it is the
 * gradient w.r.t. the last encoder layer's pre-activation, without a separate pass over the N x p*F tensor. */
int cape_gemm_ex(cape_topology* t, int M, int N, int K,
                 const float* a, int64_t a_rs, int64_t a_cs,
                 const float* b, int64_t b_rs, int64_t b_cs,
                 float* c, int64_t c_rs,
                 const float* bias, int act, float leaky_alpha, float alpha, float beta,
                 int epilogue, float epi_alpha, const float* aux, int64_t aux_rs, void* stream);

/* Many small products in ONE launch: C_i = alpha_i * A_i.B_i (beta_i = 0) or C_i += alpha_i * A_i.B_i (beta_i = 1:
 * atomic, several items may add into the same C).  The bias / condition-channel gradients of a training step are ~80
 * products of [64 x 64]-sized operands; the step's schedule is static, so the caller collects them, builds the device
 * table once (items_host != NULL: synchronous upload into table_device, n * cape_gemm_item_bytes() bytes) and from then
 * on launches it with items_host == NULL. */
typedef struct {
  const float* a; int64_t a_rs, a_cs;
  const float* b; int64_t b_rs, b_cs;
  float* c; int64_t c_rs;
  int M, N, K;
  float alpha, beta;
} cape_gemm_item;
int cape_gemm_batch(const cape_gemm_item* items_host, int n, void* table_device, int blocks_per_item, void* stream);
int cape_gemm_item_bytes(void);

/* Stand-alone mesh resampling y[n, :, :F] = S x[n, :, :F] (poolwT, lib/models.py:129-152) for an operator registered
 * in the topology (D: row selection, U: 3-tap barycentric; op < 0: identity copy); rows of x / y are x_stride /
 * y_stride floats apart.  If cond != NULL the condition channels of the reference's concat-then-unpool are written
 * as well: y[n, r, F + c] = rowsum(S)[r] * cond[n, c] (lib/models.py:606-609,750).  Backward: same call with S^T. */
int cape_resample(cape_topology* t, int op, const float* x, int x_stride, float* y, int y_stride, int N, int rows_out,
                  int rows_in, int F, const float* cond, int C, void* stream);

/* Weight re-layout for the data-gradient pass of chebyshev5: wt[(c*K + k)*Fin + f] = w[(f*K + k)*Fout + c]
 * for f < Fin (rows of w beyond Fin*K -- the condition channels -- are not touched). */
int cape_cheb_weight_transpose(const float* w, int Fin, int K, int Fout, float* wt, void* stream);

/* The derived weight layouts of MANY layers in one launch (run after every optimiser step).  Per descriptor, from the
 * reference layout w[(f*K + k)*Fout + c] (rows f < Fin; condition rows beyond are not touched):
 *   wt[(k*Fout + c)*Fin + f]   -- per-order K-major copies: tensor-core B operand of the forward pass (and, read as
 *                                 [(k, c), f], of the contract-first form Z = X @ [W_0 | W_1 | ...]), fp32-pipe operand of
 *                                 the data-gradient pass;
 *   wk[(k*Fin + f)*Fout + c]   -- per-order plain copies: K-major B operand of the contract-first data gradient
 *                                 Z = G @ [W_0^T | W_1^T | ...].
 * NULL outputs are skipped.  `descs_device`
 * is a DEVICE array of n descriptors (the pointers never change, so the caller uploads it once). */
typedef struct {
  const float* w;
  int Fin, K, Fout;
  float* wt;
  float* wk;
} cape_wprep;
int cape_weight_prep(const cape_wprep* descs_device, int n, int blocks_per_desc, void* stream);

/* ---- elementwise helpers ------------------------------------------------------------------------ */
/* g = dy * (y > 0 ? 1 : alpha)   (backward of leaky_relu given its output) */
int cape_act_bwd(const float* dy, const float* y, float* g, int64_t n, float alpha, void* stream);
/* y += a * x */
int cape_axpy(float* y, const float* x, float a, int64_t n, void* stream);
/* z = mean + sqrt(exp(logvar)) * eps  (vae_sampling, lib/models.py:193-196); z written with row stride z_stride */
int cape_vae_sample_fwd(const float* mean, const float* logvar, const float* eps, float* z, int z_stride,
                        int N, int nz, void* stream);
/* dmean = dz + kl_scale*mean/N ; dlogvar = dz*eps*0.5*sqrt(exp(lv)) + kl_scale*0.5*(exp(lv)-1)/N */
int cape_vae_sample_bwd(const float* dz, int dz_stride, const float* mean, const float* logvar, const float* eps,
                        float* dmean, float* dlogvar, int N, int nz, float kl_scale, void* stream);

/* ---- input pipeline -------------------------------------------------------------------------------
 * dst[i, 0:row_floats] = src[idx[i], 0:row_floats] for i < n: assembles a training batch from a dataset that lives in
 * HBM (replaces the numpy fancy-indexing + feed_dict of lib/models.py:877-903; only the indices cross PCIe).
 * idx is a DEVICE array; out-of-range indices are clamped. */
int cape_gather_rows(const float* src, int64_t row_floats, int n_src, const int32_t* idx_device, int n, float* dst,
                     void* stream);

/* ---- losses (CAPE.loss, lib/models.py:354-416; losses.edge_loss_calc, lib/losses.py:9-25) ----------
 * Reconstruction L1 (mean |pred-gt|; cape_recon_losses_ex below: L2 / Huber), edge loss (mean over edges of ||(p_a-p_b)-(g_a-g_b)||_2; the
 * template added at models.py:375 cancels), KL (mean_n -0.5*sum(1+lv-mu^2-e^lv)); writes
 * losses[0..2] = {recon, edge, kl} (unweighted) and ACCUMULATES lambda-weighted gradients into dpred.
 * nbr_op: id of the level-0 adjacency operator (its idx table lists each vertex's neighbours). */
int cape_recon_losses(cape_topology* t, int nbr_op, const float* pred, const float* gt, int N, int rows,
                      float lambda_l1, float lambda_edge, int n_edges,
                      const float* mean, const float* logvar, int nz,
                      float* dpred, float* losses, void* stream);
/* The reconstruction term of the reference's `--loss` switch (models.py:357-369, every one Reduction.MEAN over the
 * N*rows*3 coordinates d = pred - gt, weights 1):
 *   CAPE_RECON_L1     mean |d|                                   (absolute_difference)   gradient sign(d) / cnt
 *   CAPE_RECON_L2     mean d^2                                   (mean_squared_error)    gradient 2 d / cnt
 *   CAPE_RECON_HUBER  mean 0.5 q^2 + delta (|d| - q), q = min(|d|, delta)   (huber_loss) gradient clamp(d, +-delta) / cnt
 * losses[0] is that term, scaled into dpred by lambda_recon; the edge and KL terms are cape_recon_losses'.
 * cape_recon_losses is kind CAPE_RECON_L1 of this call (bit-identical results).  delta is read by HUBER only (> 0). */
enum { CAPE_RECON_L1 = 0, CAPE_RECON_L2 = 1, CAPE_RECON_HUBER = 2 };
int cape_recon_losses_ex(cape_topology* t, int nbr_op, const float* pred, const float* gt, int N, int rows,
                         int kind, float delta, float lambda_recon, float lambda_edge, int n_edges,
                         const float* mean, const float* logvar, int nz, float* dpred, float* losses, void* stream);
/* cape_recon_losses_ex with per-vertex weights on the reconstruction term: the reference's `--loss_mask binary`
 * (models.py:47-52 builds weights [N, rows, 1] from one per-vertex mask, :357-369 hands them to every loss kind).
 * vweight: device [rows], m[v]; vweight_sum: sum_v m[v] (> 0).  TF-1 Reduction.MEAN divides the weighted sum by the
 * sum of the weights broadcast to [N, rows, 3]:
 *   losses[0] = sum_{n,v,c} m[v] l(d) / (3 N vweight_sum),  dpred += lambda_recon m[v] l'(d) / (3 N vweight_sum)
 * with l, l' those of `kind`.  The edge and KL terms are cape_recon_losses_ex's, unweighted.  An all-ones vweight
 * (sum rows) gives bit-identical results to cape_recon_losses_ex. */
int cape_recon_losses_w(cape_topology* t, int nbr_op, const float* pred, const float* gt, int N, int rows,
                        int kind, float delta, float lambda_recon, float lambda_edge, int n_edges,
                        const float* vweight, double vweight_sum,
                        const float* mean, const float* logvar, int nz, float* dpred, float* losses, void* stream);
/* Sigmoid cross-entropy with a constant label (tf.nn.sigmoid_cross_entropy_with_logits, models.py:387-389):
 * loss[0] += mean(bce(logits, label)); dlogits = scale * d mean(bce)/dlogits  */
int cape_bce_logits(const float* logits, int64_t n, float label, float scale, float* dlogits, float* loss,
                    void* stream);

/* ---- optimiser (CAPE.training, lib/models.py:419-474) -----------------------------------------------
 * sumsq[0] += sum(g^2) (zero it first), reduced in a fixed order: bit-identical on every replica and in every run
 * (calls on one device must be ordered: they share a small scratch in device memory);  then
 * coef = clip / max(sqrt(sumsq), clip) (tf.clip_by_global_norm), a = momentum*a + coef*g, w -= lr*a
 * (tf.train.MomentumOptimizer, non-Nesterov).  lr is read from device memory (no host sync). */
int cape_sumsq(const float* g, int64_t n, float* sumsq, void* stream);
int cape_sgd_clip_update(float* w, const float* g, float* mom, int64_t n, const float* sumsq, float clip_norm,
                         const float* lr_dev, float momentum, void* stream);

/* tf.train.AdamOptimizer (the reference's `optimizer: adam` branch, lib/models.py:449-451; TF-1.13 defaults
 * beta1 = 0.9, beta2 = 0.999, eps = 1e-8) behind the same global-norm clip:
 *   g' = coef g;  m = beta1 m + (1 - beta1) g';  v = beta2 v + (1 - beta2) g'^2;  w -= lr_t m / (sqrt(v) + eps)
 * lr_t = lr sqrt(1 - beta2^t) / (1 - beta1^t) (t = applications so far + 1) is computed by the caller and read from
 * device memory, so the launch is CUDA-graph capturable like the momentum update. */
int cape_adam_clip_update(float* w, const float* g, float* m, float* v, int64_t n, const float* sumsq, float clip_norm,
                          const float* lr_t_dev, float beta1, float beta2, float eps, void* stream);

/* ---- TensorBoard summaries (CAPE.fit's FileWriter, lib/models.py:868,919-922) --------------------------------------
 * cape_histogram replaces tf.summary.histogram (lib/models.py:219,226) as TF-1.13's HistogramSummary evaluates it,
 * for many variables in one launch.  segs: device array of nseg segments (views of the parameters); limits: device
 * [nlim] ascending bucket limits, the last one DBL_MAX.  Every value is compared in double; for segment s:
 *   counts[s, b] = #{x finite : b = upper_bound(limits, x)}  (limits[b-1] <= x < limits[b])
 *   stats[s, :] = min, max, num, sum, sum of squares of its finite values, in double (min = DBL_MAX, max = -DBL_MAX
 *   when there is none); nonfinite[s] = number of NaN / Inf values (TF refuses those: "Nan in summary histogram").
 * The double sums are reduced in a fixed order: two calls give identical bits.  Uses the topology workspace
 * (1796 bytes per segment); calls on one handle must be ordered. */
typedef struct {
  const float* p;
  int64_t n;
} cape_hist_segment;
int cape_histogram(cape_topology* t, const cape_hist_segment* segs, int nseg, const double* limits, int nlim,
                   double* stats, int64_t* nonfinite, int64_t* counts, void* stream);
/* The moving averages of the loss totals (tf.train.ExponentialMovingAverage(decay).apply([loss_g, loss_d]),
 * lib/models.py:393-414, zero_debias off), advanced once per optimiser application.  losses: the step's loss buffer
 * (recon, edge, kl, gan_g, gan_d_real, gan_d_fake); fc_sumsq: sum of W^2 over the generator's regularised dense
 * kernels (cape_sumsq).  In fp32, each operation rounded on its own, left to right as the reference writes them:
 *   reg_g  = r * (r * (fc_sumsq * 0.5))                                    (r * sum_W r * l2_loss(W))
 *   loss_g = gan_g * l_gan + recon * l_recon + 0 + edge * l_edge + kl * l_latent + reg_g
 *   loss_d = (gan_d_real + gan_d_fake) * l_gan + 0
 *   shadow[i] -= (shadow[i] - loss_i) * (1 - decay)
 * One thread; no host synchronisation. */
int cape_loss_ema(const float* losses, const float* fc_sumsq, float lambda_gan, float lambda_recon, float lambda_edge,
                  float lambda_latent, float regularization, float decay, float* shadow, void* stream);

/* ---- group norm (CAPE.gn, lib/models.py:681-712) + ReLU, for the non-affine decoder blocks ------------
 * x: [N, rows, C], G groups of C/G contiguous channels; stats over (C/G x rows) per (n, g), biased variance,
 * y = relu(gamma*(x-mean)*rstd + beta).  stats: [N, G, 2] = (mean, rstd), saved for the backward pass.
 * Backward: dy is the gradient w.r.t. y (after the ReLU); dgamma/dbeta are ACCUMULATED (zero them first); dx is
 * overwritten, or added to when accumulate_dx != 0 (residual branches meeting at the block input).
 * Both use the topology workspace (N*G*2 doubles) for fp64 group sums. */
int cape_gn_relu_fwd(cape_topology* t, const float* x, int N, int rows, int C, int G, float eps,
                     const float* gamma, const float* beta, float* y, float* stats, void* stream);
int cape_gn_relu_bwd(cape_topology* t, const float* x, const float* y, const float* dy, int N, int rows, int C, int G,
                     const float* gamma, const float* stats, float* dx, int accumulate_dx, float* dgamma, float* dbeta,
                     void* stream);

/* ---- SMPL posing (demo_full's pose_result, demos.py:249-331: smplx.lbs with zero betas) -----------------------------
 * A device-resident SMPL body model with the template replaced per call, as the reference does: every mesh verts[n] is
 * posed with pose[n] (24 axis-angle vectors, global orientation first):
 *   J = J_regressor . verts[n]  (joints of the given mesh),  R_j = Rodrigues(pose[n, j]),
 *   v_posed = verts[n] + (R_1..23 - I) . posedirs,  G_j = G_parent(j) . [R_j | J_j - J_parent(j)],
 *   out[n, v] = sum_j weights[v, j] (G_j - G_j . [J_j, 0]) . [v_posed, 1].
 * cape_smpl_create copies the model to `device`: J_regressor as CSR (jreg_ptr [25], jreg_col / jreg_val [jreg_ptr[24]],
 * columns < V), posedirs [207, V * 3] (element (p, 3 v + c) = the pickle's posedirs[v, c, p]), weights [V, 24] (kept as
 * each vertex's non-zero entries) and parents [24] (parents[0] = -1, 0 <= parents[j] < j).  cape_smpl_pose takes fp32
 * device tensors verts / out [N, V, 3] and pose [N, 72], and scratch of cape_smpl_workspace_bytes(s, N) bytes
 * (16-byte aligned).  Three launches on `stream`; the pose-blend product runs on cape_gemm. */
typedef struct cape_smpl cape_smpl;
int cape_smpl_create(int device, int V, const int32_t* jreg_ptr, const int32_t* jreg_col, const float* jreg_val,
                     const float* posedirs, const float* weights, const int32_t* parents, cape_smpl** out);
void cape_smpl_destroy(cape_smpl* s);
int64_t cape_smpl_workspace_bytes(const cape_smpl* s, int N);
int cape_smpl_pose(cape_smpl* s, int N, const float* verts, const float* pose, float* out, void* workspace,
                   int64_t workspace_bytes, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* CAPE_B200_H */
