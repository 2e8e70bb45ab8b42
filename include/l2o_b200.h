/*
 * l2o_b200 — C-ABI of the H100-native (sm_90a) coordinate-wise LSTM learned-optimizer engine.
 *
 * The reference (VITA-Group/Open-L2O, L2O-DM / L2O-RNNProp) is pure Python/TensorFlow and has no
 * FFI; the seam this library sits behind is the reference's own operator surface.  Each entry point
 * cites the reference code it replaces (DM/ = "Model_Free_L2O/L2O-DM and L2O-RNNProp/"):
 *
 *   l2o_net_create / l2o_net_destroy    networks.factory + StandardDeepLSTM.__init__   DM/networks.py:34-44,157-205
 *   l2o_theta_count / l2o_theta_layout  snt.get_variables_in_module order              DM/networks.py:47-62
 *   l2o_state_floats                    Network.initial_state_for_inputs               DM/networks.py:234-236,273-276
 *   l2o_workspace_bytes                 the loop-carried tensors + TensorArray of the while_loop  DM/meta.py:361-376
 *   l2o_step                            delta, state' = net(g, state)  (one time step) DM/networks.py:207-232,254-271,287-300
 *                                       + RNNProp Adam features                        DM/meta_rnnprop_train.py:383-388
 *                                       + x_next = x + delta                           DM/meta.py:352-353
 *   l2o_unroll_fwd                      the tf.while_loop body x T                     DM/meta.py:338-376
 *                                       imitation unroll                               DM/meta_dm_train.py:463-480
 *   l2o_unroll_bwd                      tf.gradients(loss, theta) through that loop    DM/meta.py:412 (BPTT; SURVEY.md App. B)
 *   l2o_unroll_bwd_carry                the same over one segment of the loop (recompute instead of
 *                                       while_loop(swap_memory=True))                 DM/meta.py:364-370
 *   l2o_adam_step                       tf.train.AdamOptimizer(lr).minimize            DM/meta.py:411-413
 *   l2o_log_and_sign                    preprocess.LogAndSign                          DM/preprocess.py:52-70
 *   l2o_lasso_grad                      problems.lasso(_fixed) loss + tf.gradients     DM/problems.py:103-175, DM/meta.py:322-329
 *   l2o_confocal_grad                   problems.confocal_microscopy_3d + tf.gradients DM/problems.py:701-956, DM/meta.py:322-329
 *   l2o_mnist_grad                      problems.mnist (batch draw + MLP) + tf.gradients DM/problems.py:254-288, DM/meta.py:322-329
 *   l2o_mnist_conv_grad                 problems.mnist_conv (batch-norm ConvNet) + tf.gradients DM/problems.py:291-347, DM/meta.py:322-329
 *   l2o_cifar_conv_grad                 problems.cifar10 (batch-norm ConvNet) + tf.gradients DM/problems.py:369-458, DM/meta.py:322-329
 *   l2o_nas_grad                        problems.NAS (batch-norm NAS cell) + tf.gradients DM/problems.py:540-634, DM/meta.py:322-329
 *   l2o_lenet_grad                      problems.LeNet (batch-norm LeNet) + tf.gradients DM/problems.py:461-537, DM/util.py:176-184
 *
 * Conventions: every pointer is a DEVICE pointer owned by the caller (PyTorch allocates); no hidden
 * allocation; `stream` is a cudaStream_t passed as void*; every entry returns 0 or a negative
 * L2O_E_* code and never throws; calls are re-entrant per (device, stream).  All tensors fp32 except
 * the accumulators `fx`, `imit_loss`, `dtheta` which are fp64 (order-independent atomics).
 *
 * Layouts (row-major, N = number of coordinates):
 *   state arena  : for layer l (size H_l):  h_l [N][H_l] then c_l [N][H_l], layers concatenated
 *                  == the reference's tuple over layers of (hidden, cell) tensors [N, H_l].
 *   theta        : flat, Sonnet variable order: [input_projection/w [n_in,F], /b [F],]
 *                  lstm_1/w_gates [F+H1,4H1], lstm_1/b_gates [4H1], lstm_2/w_gates [H1+H2,4H2],
 *                  lstm_2/b_gates [4H2], linear/w [top,1], linear/b [1]; gate column order i|j|f|o.
 *   sequences    : [T][N] time-major; RNNProp feature sequences [T][2][N] (m~ then g~).
 *   ckpt         : [T+1] state arenas; slot t = state BEFORE step t; slot T = final state.
 */
#ifndef L2O_B200_H_
#define L2O_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define L2O_OK 0
#define L2O_E_INVALID (-1)      /* bad argument (NULL where required, n<0, T<0 ...) */
#define L2O_E_UNSUPPORTED (-2)  /* net shape / mode not compiled into this build */
#define L2O_E_CUDA (-3)         /* CUDA runtime error (see l2o_last_cuda_error) */
#define L2O_E_NOMEM (-4)

#define L2O_PRE_IDENTITY 0 /* tf.identity            DM/networks.py:188,221 */
#define L2O_PRE_LOGSIGN 1  /* preprocess.LogAndSign  DM/preprocess.py:42-70 */
#define L2O_PRE_FC 2       /* Linear(dim)+ELU        DM/networks.py:180-183,219 */

#define L2O_OPT_NONE 0
#define L2O_OPT_RASTRIGIN_SEP 1  /* f = fscale*sum(0.5(x-a)^2 - alpha*b*cos(2 pi x) + alpha)   DM/problems.py:177-213, A=I */
#define L2O_OPT_QUADRATIC_DIAG 2 /* f = fscale*sum((a*x-b)^2)                                   DM/problems.py:73-101, W diagonal */
#define L2O_OPT_QUADRATIC_BATCH 3 /* f = fscale*sum_b ||W_b x_b - y_b||^2, dense W_b [d,d] per group of d = opt_group
                                     consecutive coordinates; opt_a = W [n/d][d][d], opt_b = y [n]; exact-fp32 engine
                                     (groups exchange x through shared memory)                   DM/problems.py:73-101 */

#define L2O_ENGINE_AUTO 0
#define L2O_ENGINE_FFMA 1   /* exact-fp32 CUDA-core kernels */
#define L2O_ENGINE_TC 2     /* tensor-core wgmma (3xTF32 error-compensated) kernels */

typedef struct l2o_net* l2o_handle;

typedef struct {
  int32_t n_layers;    /* 0, 1 or 2 */
  int32_t hidden[2];   /* LSTM sizes */
  int32_t preprocess;  /* L2O_PRE_* */
  int32_t n_in;        /* 1: net(g, s) ; 2: RNNprop net(m~, g~, s) */
  int32_t fc_dim;      /* L2O_PRE_FC: projection width */
  float logsign_k;     /* L2O_PRE_LOGSIGN */
  float scale;         /* output scale                DM/networks.py:229-232 */
  int32_t tanh_output; /* 1: tanh(linear)*scale       DM/networks.py:229-230 */
} l2o_net_desc;

typedef struct {
  int64_t n;
  const float* theta;
  const float* in0;     /* [n] g (or m~ when n_in==2 and m==NULL) */
  const float* in1;     /* [n] g~ (n_in==2, operator surface) or NULL */
  float* m;             /* [n] in/out Adam first moment: non-NULL selects the fused RNNProp feature mode */
  float* v;             /* [n] in/out */
  float beta1, beta2;
  float p;              /* float(step + t)            DM/meta_rnnprop_train.py:384,386 */
  const float* state_in;/* state arena */
  float* state_out;     /* may alias state_in */
  float* x;             /* optional [n], x += delta */
  float* delta;         /* optional [n] */
  float* feat_out;      /* optional [2][n]: (m~, g~) actually fed to the net (recorded for BPTT) */
  const int32_t* step_ptr; /* optional DEVICE scalar: when non-NULL, p = float(*step_ptr + t_offset) (CUDA-graph friendly) */
  int32_t t_offset;
  int32_t reuse_weights;   /* 1: theta is unchanged since this handle's previous l2o_step / forward launch on this stream:
                              the tensor-core engine skips rebuilding its weight image (one tiny launch per step saved;
                              the caller steps T times per unroll with the same theta).  0 is always safe. */
} l2o_step_args;

typedef struct {
  int64_t n;
  int32_t T;
  const float* theta;
  const float* in_seq;  /* [T][n_in][n] pre-recorded net inputs, or NULL when opt_kind != NONE */
  int32_t opt_kind;     /* L2O_OPT_*: gradient evaluated in-kernel from x */
  const float* opt_a;
  const float* opt_b;
  float opt_alpha;
  float opt_fscale;
  float* x;             /* [n] in/out (required for in-kernel optimizees; optional otherwise) */
  float* state;         /* state arena in/out (S_0 -> S_T) */
  float* ckpt;          /* optional [T+1] arenas: slots 0..T written (slot 0 = S_0 copy) */
  float* m;             /* fused RNNProp feature mode (with opt_kind != NONE or in_seq = raw g [T][n]) */
  float* v;
  float beta1, beta2;
  int32_t step0;        /* p = float(step0 + t)       DM/util.py:59-60 */
  float* g_rec;         /* optional [T+1][n]: raw gradients g_0..g_T (g_T at x_T) for the lambda suffix sums */
  float* feat_rec;      /* optional [T][2][n]: (m~, g~) per step */
  double* fx;           /* optional [T+1]: fx[t] += f(x_t) (in-kernel optimizees) */
  float* delta_seq;     /* optional [T][n] */
  const float* labels;  /* optional [T][n]: imitation targets      DM/meta_dm_train.py:472-475 */
  double* imit_loss;    /* += sum_t 0.5*sum((label-delta)^2)/n_total */
  int64_t n_total;
  int32_t opt_group;    /* L2O_OPT_QUADRATIC_BATCH: coordinates per dense group (1..128, n % opt_group == 0) */
} l2o_unroll_args;

typedef struct {
  int64_t n;
  int32_t T;
  const float* theta;
  const float* in_seq;  /* [T][n_in][n] what the net was fed (g_rec rows 0..T-1, feat_rec, or the imitation inputs) */
  const float* ckpt;    /* [T+1] arenas (slots 0..T-1 read), 16-byte aligned (L2O_E_INVALID otherwise) */
  const float* g_rec;   /* [T+1][n] raw gradients -> dDelta_t = sum_{tau>t} g_tau ; NULL in imitation mode */
  const float* labels;  /* imitation mode: dDelta_t = (delta_t - label_t)/n_total */
  int64_t n_total;
  double* dtheta;       /* [P] += dL/dtheta */
  const float* delta_seq; /* optional [T][n], imitation mode: the deltas l2o_unroll_fwd recorded for this unroll; lets the
                             tensor-core BPTT form dDelta_t without recomputing the output layer (exact-fp32 engine ignores it) */
  float* scratch;       /* optional [T][n][20] floats, fc(20) nets (RNNProp) only: hand-over buffer between the layer-2 and the
                             layer-1 pass of the tensor-core BPTT; NULL keeps such a net on the exact-fp32 engine */
} l2o_bwd_args;

int l2o_net_create(l2o_handle* out, const l2o_net_desc* desc);
void l2o_net_destroy(l2o_handle h);
int l2o_net_set_engine(l2o_handle h, int32_t engine);
int64_t l2o_theta_count(l2o_handle h);
int64_t l2o_state_floats(l2o_handle h); /* per coordinate: 2*sum(H_l) */
/* Caller-owned buffer sizes (bytes) for n coordinates and an unroll of T steps (SURVEY.md 8(b): l2o_workspace_bytes).
 * fwd_bytes: state arena + [T+1] checkpoint arenas + g_rec [T+1][n] + feat_rec [T][2][n] (n_in == 2 only);
 * bwd_bytes: what l2o_unroll_bwd reads of those (ckpt + g_rec/in_seq) + the fp64 dtheta accumulator.
 * The library itself allocates nothing per call (only a per-net weight image of < 100 KB at first tensor-core use). */
int l2o_workspace_bytes(l2o_handle h, int64_t n, int32_t T, size_t* fwd_bytes, size_t* bwd_bytes);

/* Boundary conditions of a BPTT sweep over one segment [t0, t1) of a longer unroll (segmented BPTT: the caller keeps
 * the state only at segment starts and recomputes each segment's checkpoints before its backward).  The sweep starts
 * from these buffers instead of dh = dc = 0, lambda = g_rec[T], and writes them back when it reaches t0; one thread
 * owns each coordinate, so the update is in place.  A zero carry over a single segment is l2o_unroll_bwd. */
typedef struct {
  float* d_state;   /* [state arena] in: adjoint of the state after the segment; out: before it (16-byte aligned) */
  float* lam;       /* [n] in: sum_{tau > t1} g_tau ; out: sum_{tau > t0} g_tau */
} l2o_bwd_carry;

int l2o_step(l2o_handle h, const l2o_step_args* a, void* stream);
int l2o_unroll_fwd(l2o_handle h, const l2o_unroll_args* a, void* stream);
int l2o_unroll_bwd(l2o_handle h, const l2o_bwd_args* a, void* stream);
/* l2o_unroll_bwd over one segment with carried boundary conditions: a->T is the segment length, a->ckpt its T + 1
 * slots, a->g_rec / in_seq / delta_seq / scratch its rows (g_rec rows t0..t1).  Meta-loss mode only: imitation
 * (a->labels) returns L2O_E_UNSUPPORTED.  Same engine choice as l2o_unroll_bwd. */
int l2o_unroll_bwd_carry(l2o_handle h, const l2o_bwd_args* a, const l2o_bwd_carry* c, void* stream);
/* Which tensor-core forward kernel l2o_unroll_fwd would run *a on, without launching anything: 1 = the full-tile
 * instantiation (DM net, in-kernel Rastrigin or diagonal quadratic, n % 64 == 0, T >= 1, plain output layer, ckpt and
 * g_rec both set or both NULL), 0 = the general one, L2O_E_UNSUPPORTED = not the tensor-core engine's call. */
int l2o_tc_fwd_variant(l2o_handle h, const l2o_unroll_args* a);
/* The tensor-core engine's weight image of theta, as the forward (with_transposed = 0: B1h | B1l | B2h | B2l) or the
 * BPTT (1: + T1h | T1l | T2h | T2l) stages it in shared memory; K-major tf32 core-matrix order, DESIGN.md §3.2.  The
 * B images hold the gate weights and biases scaled by -log2e (i, f, o) and -2 log2e (j), with the forget bias +1 in
 * the bias row; the T images hold them unscaled.  img NULL: nothing is launched.  Returns the image's float count,
 * or a negative status. */
int64_t l2o_tc_weight_image(l2o_handle h, const float* theta, float* img, int32_t with_transposed, void* stream);

/* TF-1.14 Adam on theta: k = 1-based step count. */
int l2o_adam_step(float* theta, const double* dtheta, float* m, float* v, int64_t n, int32_t k, float lr,
                  float beta1, float beta2, float eps, void* stream);

/* out [2][n]: row 0 = max(log(|g|+eps)/k, -1), row 1 = clip(g*e^k, -1, 1). */
int l2o_log_and_sign(const float* g, float* out, int64_t n, float k, void* stream);

/* ---------------------------------------------------------------------------------------------------------------
 * Row-wise dense LSTM net with run-time shapes: StandardDeepLSTM with output_size > 1 = the reference's KernelDeepLSTM
 * (DM/networks.py:154-236,303-351).  A convolution kernel [kw,kh,cin,cout] is R = cin*cout rows of K = kw*kh inputs;
 * with the variable flat in its own order, element (k, r) sits at k*R + r.  theta: lstm_1/w_gates [F+H1,4H1], b_gates,
 * lstm_2/..., linear/w [top, n_out], linear/b [n_out] (F = n_in, or 2*n_in interleaved (log, sign) with LogAndSign);
 * state arena per layer: h [R][H] then c [R][H]; sequences [T][n_in][R]; g_rec [T+1][n_out][R].
 *
 *   l2o_dense_create / destroy / theta_count / state_floats   KernelDeepLSTM.__init__            DM/networks.py:311-323
 *   l2o_dense_step        update, state' = net(kernel_gradient, state)  (+ x += update)          DM/networks.py:329-346
 *   l2o_dense_unroll_bwd  tf.gradients through the unroll for this net (SURVEY.md App. B)         DM/meta.py:412 */
typedef struct l2o_dense* l2o_dense_handle;
typedef struct {
  int32_t n_layers;    /* 0, 1 or 2 */
  int32_t hidden[2];   /* <= 32 */
  int32_t n_in;        /* K raw inputs per row (<= 64 with LogAndSign, <= 128 without) */
  int32_t preprocess;  /* L2O_PRE_IDENTITY | L2O_PRE_LOGSIGN */
  float logsign_k;
  int32_t n_out;       /* outputs per row (<= 64) */
  float scale;
  int32_t tanh_output;
} l2o_dense_desc;
typedef struct {
  int64_t rows;
  const float* theta;
  const float* in;       /* [n_in][rows] */
  const float* state_in;
  float* state_out;      /* may alias state_in */
  float* x;              /* optional [n_out][rows]: x += update */
  float* delta;          /* optional [n_out][rows] */
} l2o_dense_step_args;
typedef struct {
  int64_t rows;
  int32_t T;
  const float* theta;
  const float* in_seq;   /* [T][n_in][rows] */
  const float* ckpt;     /* [T+1] state arenas, slot t = state BEFORE step t */
  const float* g_rec;    /* [T+1][n_out][rows]: dUpdate_t = sum_{tau>t} g_tau ; NULL in imitation mode */
  const float* labels;   /* imitation mode [T][n_out][rows] */
  int64_t n_total;
  double* dtheta;        /* [P] += */
} l2o_dense_bwd_args;
int l2o_dense_create(l2o_dense_handle* out, const l2o_dense_desc* desc);
void l2o_dense_destroy(l2o_dense_handle h);
int64_t l2o_dense_theta_count(l2o_dense_handle h);
int64_t l2o_dense_state_floats(l2o_dense_handle h);   /* per ROW: 2*sum(H_l) */
int l2o_dense_step(l2o_dense_handle h, const l2o_dense_step_args* a, void* stream);
int l2o_dense_unroll_bwd(l2o_dense_handle h, const l2o_dense_bwd_args* a, void* stream);

/* ---------------------------------------------------------------------------------------------------------------
 * Fused gradient producers (SURVEY.md 8(f) row 4): f and df/dx of a synthetic optimizee family in ONE launch, replacing
 * the ~15 TF ops + tf.gradients of the reference's graph (DM/problems.py:103-175, DM/meta.py:322-329).
 *
 *   l2o_lasso_grad   problems.lasso / lasso_fixed:  f = mean_b(0.5 ||A_b x_b - y_b||^2 + l1 ||x_b||_1)
 *                    g = dF/dx;  with `scale` (random-scaling trick, DM/meta_dm_train.py:336-338,384-385) the loss is
 *                    evaluated at x (.) scale and g is multiplied by scale. */
typedef struct {
  int32_t batch, m, n;  /* A [batch][m][n], y [batch][m], x [batch][n] (row-major) */
  const float* A;
  const float* y;
  const float* x;
  const float* scale;   /* optional [batch][n] */
  float l1;
  float* g;             /* [batch][n] */
  double* f;            /* optional scalar: += f */
} l2o_lasso_args;
int l2o_lasso_grad(const l2o_lasso_args* a, void* stream);

/*   l2o_confocal_grad  problems.confocal_microscopy_3d (inference=False), DM/problems.py:701-956 + tf.gradients at
 *                      DM/meta.py:322-329:  f = mean_b sum_v (sum_p psf(theta_p; v) + bg_b - t_b[v])^2 with the target
 *                      t_b = l2_normalize_v(sum_p psf(sim_p; v) + bg_sim_b), g = df/dx.  theta = x (.) scale (optional,
 *                      random-scaling trick as l2o_lasso_grad), mapped through tfd.Uniform(lo, hi).quantile(p) =
 *                      lo + p (hi - lo): I0 in [0.5, 2], x0/y0/z0 in [0.5, roi - 1], sigma_xy and sigma_z in [2, 4].
 *                      Layout of x, scale, sim and g: [6P+1][batch], rows I, x0, y0, z0, sigma_xy, sigma_z of point
 *                      0..P-1 then bg (the reference's creation order).  One CTA per batch row holds the whole image
 *                      in shared memory: 4 (V + 4 P (nx+ny+nz) + 2P) bytes, V = nx ny nz, at most 200 KB (32^3 fits
 *                      for P <= 47), L2O_E_UNSUPPORTED beyond. */
typedef struct {
  int32_t batch, num_points;
  int32_t roi[3];       /* image size nx, ny, nz */
  const float* x;       /* [6P+1][batch] */
  const float* sim;     /* [6P+1][batch] simulated parameters (and bg_sim) */
  const float* scale;   /* optional [6P+1][batch] */
  float* g;             /* [6P+1][batch] */
  double* f;            /* optional scalar: += f */
} l2o_confocal_args;
int l2o_confocal_grad(const l2o_confocal_args* a, void* stream);

/*   l2o_mnist_grad  problems.mnist, DM/problems.py:254-288 + tf.gradients at DM/meta.py:322-329:
 *                   f = mean_b xent(MLP(images[idx_b] * fp32(1/255)), labels[idx_b]) with a fresh batch of `batch`
 *                   indices idx_b drawn uniformly from [0, num_examples) at every call (the reference's
 *                   tf.random_uniform + tf.gather), g = df/dx.  The draw is Philox4x32-10 keyed by `seed` at the
 *                   device counter *counter, which the call reads and advances by one; idx_b = (r * N) >> 32 of the
 *                   32-bit draw r (bias at most N / 2^32).  x, scale and g are the arena of the MLP's variables in
 *                   creation order: w0 [784][h0], b0 [h0], w1 [h0][h1], b1, ..., w_L [h_last][10], b_L [10].  Sigmoid
 *                   or ReLU between layers, none after the last; theta = x (.) scale (optional, random-scaling trick as
 *                   l2o_lasso_grad).  One thread-block cluster; deterministic (no atomics).  Limits: 1..4 hidden layers
 *                   of width 1..64 and batch 1..1024; anything else is L2O_E_INVALID. */
#define L2O_MNIST_INPUT 784
#define L2O_MNIST_CLASSES 10
#define L2O_MNIST_MAX_HIDDEN 4
#define L2O_MNIST_MAX_WIDTH 64
#define L2O_MNIST_MAX_BATCH 1024
#define L2O_MNIST_SIGMOID 0
#define L2O_MNIST_RELU 1
typedef struct {
  int32_t batch;          /* B */
  int32_t num_examples;   /* N: rows of images / labels */
  int32_t n_layers;       /* linear layers: hidden layers + 1 */
  int32_t hidden[4];      /* widths of the hidden layers */
  int32_t activation;     /* L2O_MNIST_SIGMOID | L2O_MNIST_RELU */
  uint64_t seed;
  int64_t* counter;       /* device scalar: read, then += 1 */
  const uint8_t* images;  /* [N][784] raw pixels */
  const uint8_t* labels;  /* [N], each < 10 */
  const float* x;         /* the arena */
  const float* scale;     /* optional, the arena's layout */
  float* g;               /* the arena's layout */
  double* f;              /* optional scalar: = f */
  int32_t* idx_out;       /* optional [B]: the indices drawn */
} l2o_mnist_args;
int l2o_mnist_grad(const l2o_mnist_args* a, void* stream);

/*   l2o_mnist_conv_grad  problems.mnist_conv(batch_norm=True), DM/problems.py:291-347 + tf.gradients at
 *                   DM/meta.py:322-329: f = mean_b xent(ConvNet(images[idx_b] * fp32(1/255)), labels[idx_b]) with a
 *                   fresh batch drawn exactly as l2o_mnist_grad draws it (same seed / counter convention, same indices),
 *                   g = df/dx.  The ConvNet (NHWC): conv 3x3 1->16 VALID + b1, batch norm, ReLU, max-pool 2x2/2;
 *                   conv 5x5 16->32 VALID + b2, batch norm, ReLU, max-pool 2x2/2 ([9,9] -> [4,4]); flatten (h, w, c);
 *                   fc 512->10 + bias, ReLU; batch norm in training mode with gamma = 1, beta = 0, eps 1e-3 and the
 *                   biased variance over all B*H*W positions.  x, scale and g are the arena of the variables in creation
 *                   order: conv_layer1/weights1 [3][3][1][16], conv_layer1/biases1 [16], conv_layer2/weights1
 *                   [5][5][16][32], conv_layer2/biases1 [32], fc_weights [512][10], fc_bias [10] (18,122 floats);
 *                   theta = x (.) scale (optional, random-scaling trick as l2o_lasso_grad).  One cooperative launch over
 *                   the resident CTAs; bitwise deterministic on any SM count (no atomics).  `workspace` is caller-owned
 *                   device memory of at least l2o_mnist_conv_workspace_bytes(batch) bytes, 16-byte aligned.  Limits:
 *                   batch 1..1024; anything else, a null required pointer, a misaligned pointer or a short workspace
 *                   is L2O_E_INVALID before any CUDA call. */
#define L2O_MNIST_CONV_COORDS 18122
#define L2O_MNIST_CONV_MAX_BATCH 1024
typedef struct {
  int32_t batch;          /* B */
  int32_t num_examples;   /* N: rows of images / labels */
  uint64_t seed;
  int64_t* counter;       /* device scalar: read, then += 1 */
  const uint8_t* images;  /* [N][784] raw pixels */
  const uint8_t* labels;  /* [N], each < 10 */
  const float* x;         /* the arena */
  const float* scale;     /* optional, the arena's layout */
  float* g;               /* the arena's layout */
  double* f;              /* optional scalar: = f */
  int32_t* idx_out;       /* optional [B]: the indices drawn */
  void* workspace;        /* caller-owned, >= l2o_mnist_conv_workspace_bytes(batch) bytes */
  size_t workspace_bytes;
} l2o_mnist_conv_args;
/* bytes of workspace l2o_mnist_conv_grad needs at this batch size; L2O_E_INVALID outside 1..1024 */
int64_t l2o_mnist_conv_workspace_bytes(int32_t batch);
/* byte offsets inside the workspace of what the last call's ReLU and max-pool decisions were made from, so that a
 * caller can check g against a reference taking the same decisions: [0] z1 (fp32 [B][26][26][16], conv1 + b1),
 * [1] z2 (fp32 [B][9][9][32], conv2 + b2), [2] bn (fp32 [96]: mu1 [16], rstd1 [16], mu2 [32], rstd2 [32]; the
 * normalised value is (z - mu) * rstd in fp32), [3] dlogits (fp32 [B][16], zero where the logit's ReLU is off).
 * L2O_E_INVALID outside 1..1024 or for a null off. */
#define L2O_MNIST_CONV_LAYOUT 4
int l2o_mnist_conv_workspace_layout(int32_t batch, int64_t* off);
int l2o_mnist_conv_grad(const l2o_mnist_conv_args* a, void* stream);

/*   l2o_cifar_conv_grad  problems.cifar10(batch_norm=True), DM/problems.py:369-458 + tf.gradients at
 *                   DM/meta.py:322-329: f = mean_b xent(ConvNet(images[idx_b] / 255), labels[idx_b]) with a fresh batch
 *                   drawn as l2o_mnist_grad draws it (same seed / counter convention; the indices are uniform over the
 *                   N rows given), g = df/dx.  A pixel is fp32(p) / fp32(255), a correctly rounded division, read NHWC
 *                   from the record's [3][32][32] planes.  The ConvNet (NHWC): conv 3x3 3->16 stride 2 VALID + b1
 *                   ([32,32] -> [15,15]), batch norm, ReLU, max-pool 2x2/2 ([15,15] -> [7,7]); conv 5x5 16->32 stride 2
 *                   VALID + b2 ([7,7] -> [2,2]), batch norm, ReLU, max-pool 2x2/2 ([2,2] -> [1,1]); the 32 channels;
 *                   fc 32->10 + bias, ReLU; batch norm in training mode with gamma = 1, beta = 0, eps 1e-3 and the
 *                   biased variance over all B*H*W positions.  x, scale and g are the arena of the variables in creation
 *                   order: conv_layer1/weights1 [3][3][3][16], conv_layer1/biases1 [16], conv_layer2/weights1
 *                   [5][5][16][32], conv_layer2/biases1 [32], fc_weights [32][10], fc_bias [10] (13,610 floats);
 *                   theta = x (.) scale (optional, random-scaling trick as l2o_lasso_grad).  One cooperative launch over
 *                   the resident CTAs; bitwise deterministic on any SM count (no atomics).  `workspace` is caller-owned
 *                   device memory of at least l2o_cifar_conv_workspace_bytes(batch) bytes, 16-byte aligned.  Limits:
 *                   batch 1..1024; anything else, a null required pointer, a misaligned pointer or a short workspace
 *                   is L2O_E_INVALID before any CUDA call. */
#define L2O_CIFAR_CONV_COORDS 13610
#define L2O_CIFAR_CONV_MAX_BATCH 1024
typedef struct {
  int32_t batch;          /* B */
  int32_t num_examples;   /* N: rows of images / labels */
  uint64_t seed;
  int64_t* counter;       /* device scalar: read, then += 1 */
  const uint8_t* images;  /* [N][3][32][32] raw pixels, the record's plane order */
  const uint8_t* labels;  /* [N], each < 10 */
  const float* x;         /* the arena */
  const float* scale;     /* optional, the arena's layout */
  float* g;               /* the arena's layout */
  double* f;              /* optional scalar: = f */
  int32_t* idx_out;       /* optional [B]: the indices drawn */
  void* workspace;        /* caller-owned, >= l2o_cifar_conv_workspace_bytes(batch) bytes */
  size_t workspace_bytes;
} l2o_cifar_conv_args;
/* bytes of workspace l2o_cifar_conv_grad needs at this batch size; L2O_E_INVALID outside 1..1024 */
int64_t l2o_cifar_conv_workspace_bytes(int32_t batch);
/* byte offsets inside the workspace of what the last call's ReLU and max-pool decisions were made from, so that a
 * caller can check g against a reference taking the same decisions: [0] z1 (fp32 [B][15][15][16], conv1 + b1),
 * [1] z2 (fp32 [B][2][2][32], conv2 + b2), [2] bn (fp32 [96]: mu1 [16], rstd1 [16], mu2 [32], rstd2 [32]; the
 * normalised value is (z - mu) * rstd in fp32), [3] dlogits (fp32 [B][16], zero where the logit's ReLU is off).
 * L2O_E_INVALID outside 1..1024 or for a null off. */
#define L2O_CIFAR_CONV_LAYOUT 4
int l2o_cifar_conv_workspace_layout(int32_t batch, int64_t* off);
int l2o_cifar_conv_grad(const l2o_cifar_conv_args* a, void* stream);

/*   l2o_nas_grad     problems.NAS(batch_norm=True), DM/problems.py:540-634 + tf.gradients at DM/meta.py:322-329:
 *                   f = mean_b xent(NAS(images[idx_b] / 255), labels[idx_b]), the batch and the pixels as
 *                   l2o_cifar_conv_grad, g = df/dx.  The network (NHWC): every conv 3x3 SAME stride 1 + bias, batch norm,
 *                   ReLU; node0 = conv(x, 3->16), n0o2 = conv(node0), node1 = conv(node0), n1o3 = conv(node1) (16->16);
 *                   node2 = avgpool 3x3/1 SAME(node1) + n0o2, the average over the in-image cells of each window;
 *                   node3 = node2 + n1o3 + node0; the mean over the 1024 positions; fc 16->10 + bias, ReLU.  Batch norm
 *                   as l2o_cifar_conv_grad.  x, scale and g are the arena of the variables in creation order:
 *                   node0/weights1 [3][3][3][16], node0/biases1 [16], then node0_onto_node2, node1 and node1_onto_node3,
 *                   each weights1 [3][3][16][16] and biases1 [16], then fc_weights [16][10], fc_bias [10] (7,578 floats).
 *                   One cooperative launch, seven grid barriers; bitwise deterministic on any SM count (no atomics).
 *                   Workspace, alignment and limits (batch 1..1024) as l2o_cifar_conv_grad. */
#define L2O_NAS_COORDS 7578
#define L2O_NAS_MAX_BATCH 1024
typedef struct {
  int32_t batch;          /* B */
  int32_t num_examples;   /* N: rows of images / labels */
  uint64_t seed;
  int64_t* counter;       /* device scalar: read, then += 1 */
  const uint8_t* images;  /* [N][3][32][32] raw pixels, the record's plane order */
  const uint8_t* labels;  /* [N], each < 10 */
  const float* x;         /* the arena */
  const float* scale;     /* optional, the arena's layout */
  float* g;               /* the arena's layout */
  double* f;              /* optional scalar: = f */
  int32_t* idx_out;       /* optional [B]: the indices drawn */
  void* workspace;        /* caller-owned, >= l2o_nas_workspace_bytes(batch) bytes */
  size_t workspace_bytes;
} l2o_nas_args;
/* bytes of workspace l2o_nas_grad needs at this batch size; L2O_E_INVALID outside 1..1024 */
int64_t l2o_nas_workspace_bytes(int32_t batch);
/* byte offsets inside the workspace of what the last call's ReLU decisions were made from: [0] z0, [1] za (n0o2),
 * [2] z1 (node1), [3] zb (n1o3), each fp32 [B][32][32][16], conv + bias before batch norm; [4] bn (fp32 [4][2][16]:
 * mu and rstd of node0, n0o2, node1, n1o3 in that order; the normalised value is (z - mu) * rstd in fp32), [5] dlogits
 * (fp32 [B][16], zero where the logit's ReLU is off).  L2O_E_INVALID outside 1..1024 or for a null off. */
#define L2O_NAS_LAYOUT 6
int l2o_nas_workspace_layout(int32_t batch, int64_t* off);
int l2o_nas_grad(const l2o_nas_args* a, void* stream);

/*   l2o_lenet_grad   problems.LeNet(conv_channels=(6, 16), linear_layers=(120, 84), batch_norm=True),
 *                   DM/problems.py:461-537 as DM/util.py:176-184 builds it, + tf.gradients at DM/meta.py:322-329:
 *                   f = mean_b xent(LeNet(images[idx_b] / 255), labels[idx_b]), the batch and the pixels as
 *                   l2o_cifar_conv_grad, g = df/dx.  The network (NHWC): conv 5x5 3->6 stride 1 VALID + b ([32,32] ->
 *                   [28,28]), batch norm + beta, sigmoid, max-pool 2x2/2 ([28,28] -> [14,14]); conv 5x5 6->16 the same
 *                   way ([14,14] -> [10,10] -> [5,5]); the (h, w, c) flatten of 400; linear 400->120 + b, batch norm
 *                   over the batch + beta, sigmoid; linear 120->84 likewise; linear 84->10 + b, no activation.  Batch
 *                   norm in training mode with no gamma, eps 1e-3 and the biased variance; its beta IS a variable.
 *                   x, scale and g are the arena of the 14 variables in creation order: conv_2d_0/w [5][5][3][6],
 *                   conv_2d_0/b [6], batch_norm_0/beta [6], conv_2d_1/w [5][5][6][16], /b [16], batch_norm_1/beta
 *                   [16], mlp/linear_0/w [400][120], /b [120], mlp/batch_norm/beta [120], linear_1/w [120][84], /b
 *                   [84], mlp/batch_norm_1/beta [84], linear_2/w [84][10], /b [10] (62,232 floats).  One cooperative
 *                   launch, eleven grid barriers; bitwise deterministic on any SM count (no atomics).  Workspace,
 *                   alignment and limits (batch 1..1024) as l2o_cifar_conv_grad. */
#define L2O_LENET_COORDS 62232
#define L2O_LENET_MAX_BATCH 1024
typedef struct {
  int32_t batch;          /* B */
  int32_t num_examples;   /* N: rows of images / labels */
  uint64_t seed;
  int64_t* counter;       /* device scalar: read, then += 1 */
  const uint8_t* images;  /* [N][3][32][32] raw pixels, the record's plane order */
  const uint8_t* labels;  /* [N], each < 10 */
  const float* x;         /* the arena */
  const float* scale;     /* optional, the arena's layout */
  float* g;               /* the arena's layout */
  double* f;              /* optional scalar: = f */
  int32_t* idx_out;       /* optional [B]: the indices drawn */
  void* workspace;        /* caller-owned, >= l2o_lenet_workspace_bytes(batch) bytes */
  size_t workspace_bytes;
} l2o_lenet_args;
/* bytes of workspace l2o_lenet_grad needs at this batch size; L2O_E_INVALID outside 1..1024 */
int64_t l2o_lenet_workspace_bytes(int32_t batch);
/* byte offsets inside the workspace of what the last call's max-pool decisions were made from: [0] z0 (fp32
 * [B][28][28][6], conv0 + b), [1] z1 (fp32 [B][10][10][16], conv1 + b), [2] bn (fp32 [452]: mu0 [6], rstd0 [6],
 * mu1 [16], rstd1 [16], then linear_0's mu [120] and rstd [120] and linear_1's mu [84] and rstd [84], as applied: the
 * normalised value is (z - mu) * rstd in fp32).  Each window's decision is the first maximum of z in row-major order
 * (batch norm, + beta and the sigmoid are increasing).  L2O_E_INVALID outside 1..1024 or for a null off. */
#define L2O_LENET_LAYOUT 3
int l2o_lenet_workspace_layout(int32_t batch, int64_t* off);
int l2o_lenet_grad(const l2o_lenet_args* a, void* stream);

/* ---------------------------------------------------------------------------------------------------------------
 * L2O-Scale HierarchicalRNN update step (SURVEY.md 8(f) row 1; BASELINE config #4).
 * SC/ = Model_Free_L2O/L2O-Scale/L2O-Scale-Training/ ; HR = SC/optimizer/hierarchical_rnn.py.
 *
 *   l2o_hrnn_create            HierarchicalRNN.__init__ + _create_slots (one slot set per optimizee tensor)   HR:69-218
 *   l2o_hrnn_init_state        _initialize_state / _initialize_global_state                                    HR:303-350
 *   l2o_hrnn_prepare           (derived quantities of a fresh / restored state: mean log-lr HR:432-442, first-step
 *                               predicate SC/optimizer/utils.py:128-130, per-tensor gate bias HR:561-575)
 *   l2o_hrnn_step              _compute_updates: one optimizer step over all tensors                          HR:353-430
 *
 * The flag set is the one the reference's drivers run (SC/metarun.py:154-225,243): levels [10,20,20], 4 gradient
 * scales, grad products, log mean-squares, relative lr against the problem-wide mean, gradient shortcut, dynamic
 * output scale, learnable decays / RNN init; no attention.  theta: flat fp32 [l2o_hrnn_theta_count()] in TF variable
 * creation order (documented in open_l2o_b200/hierarchical_rnn.py THETA_SPEC).  state: 21 fp32 planes of [N]
 * (N = sum of tensor sizes, tensors contiguous): 0-9 parameter (hidden), 10 scl_decay, 11 inp_decay,
 * 12 log_learning_rate, 13-16 grad_accum1..4, 17-20 ms1..4.  layer: [n_tensors][20]; global: [20].
 * workspace: caller-owned device buffer of l2o_hrnn_workspace_bytes() bytes, 256-byte aligned; it carries the
 * per-tensor reductions from one step to the next, so it belongs to the state (call l2o_hrnn_prepare after writing
 * the state from outside). */
typedef struct l2o_hrnn* l2o_hrnn_handle;
typedef struct {
  const float* theta;
  float* x;         /* [N] optimizee parameters, updated in place (not needed by init_state / prepare) */
  const float* g;   /* [N] gradients */
  float* state;     /* [21][N] */
  float* layer;     /* [n_tensors][20] per-tensor RNN states */
  float* global;    /* [20] global RNN state */
  void* workspace;
  float* update;    /* optional [N]: the applied step (x_old - x_new) */
} l2o_hrnn_args;
int l2o_hrnn_create(l2o_hrnn_handle* out, const int64_t* tensor_sizes, int32_t n_tensors);
void l2o_hrnn_destroy(l2o_hrnn_handle h);
int64_t l2o_hrnn_theta_count(void);
int64_t l2o_hrnn_state_floats(void);           /* 21 per coordinate */
int64_t l2o_hrnn_coords(l2o_hrnn_handle h);    /* N */
int64_t l2o_hrnn_workspace_bytes(l2o_hrnn_handle h);
int l2o_hrnn_init_state(l2o_hrnn_handle h, const l2o_hrnn_args* a, void* stream); /* all planes but log_learning_rate */
int l2o_hrnn_prepare(l2o_hrnn_handle h, const l2o_hrnn_args* a, void* stream);
int l2o_hrnn_step(l2o_hrnn_handle h, const l2o_hrnn_args* a, void* stream);
/* Sharded use (SURVEY.md 8(e): the one path with an exchange per INNER step).  Every rank holds a contiguous slice of
 * every tensor's coordinates (tensor_sizes given to l2o_hrnn_create are the LOCAL counts, 0 allowed) and replicas of
 * layer / global.  l2o_hrnn_set_global_sizes gives the counts the per-tensor and problem-wide means divide by.  Per
 * step: l2o_hrnn_step_local; all-reduce SUM of the n_tensors x 24 fp64 sums at workspace offset [0] and all-reduce MAX
 * of the n_tensors x 4 int32 flags at offset [1] (l2o_hrnn_workspace_layout); l2o_hrnn_step_finish.  Same for
 * prepare.  l2o_hrnn_step / l2o_hrnn_prepare are exactly local + finish. */
int l2o_hrnn_set_global_sizes(l2o_hrnn_handle h, const int64_t* global_sizes);
int l2o_hrnn_prepare_local(l2o_hrnn_handle h, const l2o_hrnn_args* a, void* stream);
int l2o_hrnn_prepare_finish(l2o_hrnn_handle h, const l2o_hrnn_args* a, void* stream);
int l2o_hrnn_step_local(l2o_hrnn_handle h, const l2o_hrnn_args* a, void* stream);
int l2o_hrnn_step_finish(l2o_hrnn_handle h, const l2o_hrnn_args* a, void* stream);

/* Meta-training of the HierarchicalRNN (SC/optimizer/trainable_optimizer.py:200-470: BPTT through the unrolled
 * optimizer).  The reference's default, use_second_derivatives=True, differentiates through the optimizee's gradients
 * g as well; it stop_gradient's them only when the flag is off (:330-338).  g is a constant of this backward when d_g
 * is null; otherwise d_g receives the adjoint of g, which the caller carries on to x through the optimizee's
 * Hessian-vector product.  The per-parameter level — everything that
 * touches N coordinates — is differentiated by l2o_hrnn_coord_bwd; the per-tensor / global GRUs, the 1/RMS(delta)
 * normalisation, the problem-wide mean log-lr and the objective are [n_tensors x 20]-sized and are differentiated by the
 * host (open_l2o_b200/hrnn_train.py builds them as torch autograd around these two entry points).
 *   forward of one step:   write bias0 / zero_flag / mean_log_lr into the workspace (l2o_hrnn_workspace_layout), zero the
 *                          sums, l2o_hrnn_step_local (planes in place, raw update lr*delta and the per-tensor sums in the
 *                          workspace);
 *   backward of that step: l2o_hrnn_coord_bwd with the planes BEFORE the step and the same per-tensor inputs. */
typedef struct {
  const float* theta;
  const float* state_old;    /* [21][N] planes before the step */
  const float* g;            /* [N] */
  const float* bias0;        /* [n_tensors][32]: injected gate bias r(10) | u(10) | c(10) | pad, as the forward step used it */
  const int32_t* zero_flag;  /* [n_tensors][4] */
  const float* mean_log_lr;  /* [1] */
  const float* d_state_new;  /* [21][N] adjoints of the planes after the step */
  const float* d_upd;        /* [N] adjoint of the raw update lr*delta (before the per-tensor 1/RMS) */
  const float* d_sums;       /* [n_tensors][24] adjoints of the per-tensor sums: h'(10) | feat(12) | delta^2 | log-lr' */
  float* d_state_old;        /* [21][N] out */
  double* d_theta;           /* [theta_count] += (the 739 per-parameter-level weights) */
  double* d_bias0;           /* [n_tensors][32] += */
  double* d_mean_log_lr;     /* [1] += */
  float* d_g;                /* optional [N] out: adjoint of g; 4-byte aligned, overlapping no other buffer (else L2O_E_INVALID) */
} l2o_hrnn_bwd_args;
int l2o_hrnn_coord_bwd(l2o_hrnn_handle h, const l2o_hrnn_bwd_args* a, void* stream);
/* byte offsets inside the workspace: [0] sums (fp64 [n_tensors][24]) [1] any_nz (int32 [n_tensors][4]) [2] zero_flag
 * (int32 [n_tensors][4]) [3] bias0 (fp32 [n_tensors][32]) [4] inv_denom (fp32 [n_tensors]) [5] mean_log_lr (fp32 [1])
 * [6] raw update (fp32 [N]) */
int l2o_hrnn_workspace_layout(l2o_hrnn_handle h, int64_t offsets[7]);

/* ---------------------------------------------------------------------------------------------------------------
 * L2O-Scale CoordinatewiseRNN (CR = SC/optimizer/coordinatewise_rnn.py): a 3-layer TF LSTMCell stack [10, 20, 20] run
 * on every coordinate independently, with learnable RMS decay and dynamic output scale.  No handle: the update has no
 * cross-coordinate term, so one step over all optimizee tensors is one launch over their concatenated coordinates.
 *
 *   l2o_crnn_theta_count   the variables of CoordinatewiseRNN.__init__ + the cells' first call        CR:80-102,206
 *   l2o_crnn_state_floats  _initialize_state: rnn [100] | rms | decay | learning_rate                  CR:151-173
 *   l2o_crnn_step          _compute_update: rms_scaling, MultiRNNCell, readouts, x - lr'*delta       CR:175-250,
 *                                                                              SC/optimizer/utils.py:108-160
 *   l2o_crnn_bwd           tf.gradients of that step (TrainableOptimizer.train BPTT).  The optimizee gradient g is a
 *                          constant when d_g is null, as in the reference with use_second_derivatives off
 *                          (SC/optimizer/trainable_optimizer.py:330-338); the reference's default differentiates
 *                          through g, and d_g then receives its adjoint
 *
 * theta: fp32 [6402] in TF variable creation order (open_l2o_b200/coordinatewise_rnn.py THETA_SPEC).  state: 103 fp32
 * planes of [n]: 0..99 the rnn slot packed c1 h1 c2 h2 c3 h3 (c before h, CR:306-315), 100 rms, 101 decay,
 * 102 learning_rate.  Every float pointer must be 4-byte aligned and d_theta 8-byte aligned (L2O_E_INVALID otherwise). */
typedef struct {
  int64_t n;               /* coordinates (> 0) */
  const float* theta;
  const float* g;          /* [n] gradients */
  const float* state_in;   /* [103][n] */
  float* state_out;        /* [103][n]; may alias state_in */
  float* x;                /* optional [n]: x -= lr' * delta */
  float* update;           /* optional [n]: lr' * delta */
} l2o_crnn_step_args;
typedef struct {
  int64_t n;
  const float* theta;
  const float* g;            /* [n] the gradients the step was fed */
  const float* state_old;    /* [103][n] planes before the step */
  const float* d_state_new;  /* [103][n] adjoints of the planes after the step */
  const float* d_update;     /* [n] adjoint of lr' * delta */
  float* d_state_old;        /* [103][n] out; must not overlap any input */
  double* d_theta;           /* [6402] += (the init_vector block is not touched: it only enters the initial state) */
  float* d_g;                /* optional [n] out: adjoint of g; 4-byte aligned, overlapping no other buffer (else L2O_E_INVALID) */
} l2o_crnn_bwd_args;
int64_t l2o_crnn_theta_count(void);
int64_t l2o_crnn_state_floats(void);
int l2o_crnn_step(const l2o_crnn_step_args* a, void* stream);
int l2o_crnn_bwd(const l2o_crnn_bwd_args* a, void* stream);

/* ---------------------------------------------------------------------------------------------------------------
 * L2O-Scale's meta-trained hand-designed baselines (SC/optimizer/): TrainableAdam (TA = trainable_adam.py),
 * LearningRateSchedule (LRS = learning_rate_schedule.py) and GlobalLearningRate (GLR = global_learning_rate.py).  No
 * handle; one launch per step and one per backward step over the concatenated coordinates of all optimizee tensors.
 *
 *   l2o_tadam_theta_count   log_learning_rate, beta1_logit, beta2_logit, log_epsilon (creation order)   TA:63-82
 *   l2o_tadam_state_floats  _initialize_state: m | t | v, zeros, in sorted key order                  TA:89-93
 *   l2o_tadam_step          _compute_update, with the reference's v' = v / (1 - pow(g^2, b2))           TA:95-175
 *   l2o_tadam_bwd           tf.gradients of that step; where v == 0 the v-chain terms are exactly 0
 *   l2o_lrsgd_step          LRS _compute_update: x - rates[min(itr, n_steps-1)] g, itr + 1             LRS:48-60
 *                           GlobalLearningRate: a one-entry table and a null itr                        GLR:38-39
 *   l2o_lrsgd_bwd           tf.gradients of that step
 * In both backward entries g is a constant when d_g is null (use_second_derivatives off,
 * SC/optimizer/trainable_optimizer.py:330-338); with d_g set it receives g's adjoint and nothing else changes.
 * theta, the schedule and the counter stay in device memory (a CUDA-graph replay needs no host synchronisation).
 * Float pointers must be 4-byte aligned, double pointers 8-byte aligned (L2O_E_INVALID otherwise). */
typedef struct {
  int64_t n;               /* coordinates (> 0) */
  const float* theta;      /* [4] */
  const float* g;          /* [n] */
  const float* state_in;   /* [3][n] m | t | v */
  float* state_out;        /* [3][n]; may alias state_in */
  float* x;                /* optional [n]: x -= update */
  float* update;           /* optional [n]: lr m^ / (sqrt(v^ + 1e-10) + eps) */
} l2o_tadam_step_args;
typedef struct {
  int64_t n;
  const float* theta;        /* [4] */
  const float* g;            /* [n] the gradients the step was fed */
  const float* state_old;    /* [3][n] planes before the step */
  const float* d_state_new;  /* [3][n] adjoints of the planes after the step (the t plane's is ignored) */
  const float* d_update;     /* [n] */
  float* d_state_old;        /* [3][n] out (the t plane gets 0); must not overlap any input */
  double* d_theta;           /* [4] += */
  float* d_g;                /* optional [n] out: adjoint of g; 4-byte aligned, overlapping no other buffer (else L2O_E_INVALID) */
} l2o_tadam_bwd_args;
typedef struct {
  int64_t n;               /* coordinates (> 0) */
  const float* rates;      /* [n_steps] the schedule (GlobalLearningRate: its one rate) */
  int32_t n_steps;         /* > 0 */
  int32_t* itr;            /* optional int32 [2]: step index, then an arrival count that is 0 between launches.  The
                              step uses rates[min(itr[0], n_steps-1)] and advances itr[0] by one in place.  Null: index 0 */
  const float* g;          /* [n] */
  float* x;                /* optional [n]: x -= update */
  float* update;           /* optional [n]: rate * g */
} l2o_lrsgd_step_args;
typedef struct {
  int64_t n;
  const float* rates;      /* [n_steps] */
  int32_t n_steps;
  const int32_t* itr;      /* optional [2]: the counter as the step saw it (before it advanced); null: index 0 */
  const float* g;          /* [n] */
  const float* d_update;   /* [n] */
  double* d_rates;         /* [n_steps] += (only the entry the step used) */
  float* d_g;              /* optional [n] out: rate * d_update; 4-byte aligned, overlapping no other buffer */
} l2o_lrsgd_bwd_args;
int64_t l2o_tadam_theta_count(void);
int64_t l2o_tadam_state_floats(void);
int l2o_tadam_step(const l2o_tadam_step_args* a, void* stream);
int l2o_tadam_bwd(const l2o_tadam_bwd_args* a, void* stream);
int l2o_lrsgd_step(const l2o_lrsgd_step_args* a, void* stream);
int l2o_lrsgd_bwd(const l2o_lrsgd_bwd_args* a, void* stream);

/* ---------------------------------------------------------------------------------------------------------------
 * Model-based L2O's LISTA family (MB = Model_Base_L2O/): ISTA unrolled into K trained layers, starting from x_0 = 0.
 * Row-major: y [B][M] (row stride ldy, so a data batch [y | x_true] can be passed as is), x [B][N], A [M][N].
 *
 *   l2o_ista_fwd              layers [k0, k1) of the Keras model's call                       MB/models/lista.py:32-45
 *                             (one launch)                                   lista_cp.py, lista_cpss.py:29-39, alista.py:29-39
 *                             with shrink_free / shrink_ss                                    MB/models/utils.py:11-52
 *   l2o_ista_bwd              tf.gradients of a loss on x_{k1} w.r.t. every variable          MB/train.py:307 (model.fit)
 *                             and x_{k0}, times utils.Adam's 0.3^age multipliers              MB/utils.py:115-135
 *                             (two launches; apply them with l2o_adam_step, eps = 1e-7 for Keras)
 *   l2o_ista_loss_grad        utils.MSE / utils.LassoLoss per row and their gradient          MB/utils.py:6-38
 *   l2o_ista_workspace_bytes  the scratch l2o_ista_bwd needs (dz_k and per-CTA partial sums)
 *
 * Forms: L2O_ISTA_LISTA   z_k = y B1^T + s_k x_k W_k^T  (layer 0 has no W term); B1 [N][M], W slots [N][N], slot k-1
 *                         for layer k (one slot when share_W).
 *        L2O_ISTA_COUPLED z_k = x_k + s_k (y - x_k A^T) W_k;  W slots [M][N], slot k (one slot when share_W).
 *        L2O_ISTA_LFISTA  z_k = y We^T + [k>=1] x_k Wg_k^T + [k>=2] x_{k-1} Wm_k^T       MB/models/lfista.py
 *                         B1 = We [N][M], W = Wg slots and W2 = Wm slots [N][N], slot k-1 for layer k; no share_W,
 *                         no step.  x_{k0-1} comes from s2_in.
 *        L2O_ISTA_LAMP    v_k = y - x_k A^T + b_k v_{k-1}, b_k = ||x_k||_0 / M (b_0 = 0),  MB/models/lamp.py
 *                         z_k = r_k = x_k + s_k v_k W_k, shrunk with the row's theta = max(sqrt(||v_k||^2 / M) lam_k,
 *                         0); theta holds lam_k.  A, W slots [M][N] as the coupled form; rs records v_k.
 *                         v_{k0-1} comes from s2_in.  The backward takes |r| >= theta (tf.maximum's tie rule) as live
 *                         and gives a row with rvar = 0 no gradient through its theta.
 * x_{k+1} = sign(z) relu(|z| - theta_k); with ss_rank, entries with |z| > theta_k and |z| > t_b pass unshrunk, t_b
 * being row b's |z| at 0-based rank ss_rank[k] in descending order (the caller maps the percentile to the rank).
 * LFISTA and LAMP take no ss_rank.  Their backward also carries the second state: d_s2 enters as its adjoint at the
 * top of the pass and d_s2_in returns it at the bottom, so passes [0, j) and [j, K) compose as one.
 * The backward overwrites every gradient it is given (zero for layers outside [k0, k1)); gscale[j] multiplies the
 * gradient of every variable created with layer j (B1: layer 0; a shared W: its first layer).  L2O_E_UNSUPPORTED when
 * M or N > 2048 or when a CTA's shared-memory plan exceeds 200 KB: 4 (8 (M + 4N) + 2048) bytes in the LISTA form,
 * 4 (8 (2M + 3N) + 2048) in the coupled and LAMP forms (so the coupled form at M = 256, N = 512 needs 72 KB and at
 * M = 1024 fits N <= 1365), 4 (8 (M + 5N) + 2048) in the LFISTA form; l2o_ista_loss_grad: 4 (M + N) bytes > 200 KB.  Float pointers 4-byte aligned, double pointers
 * 8-byte aligned (L2O_E_INVALID otherwise). */
#define L2O_ISTA_LISTA 0
#define L2O_ISTA_COUPLED 1
#define L2O_ISTA_LFISTA 2
#define L2O_ISTA_LAMP 3
#define L2O_ISTA_TASK_SC 0
#define L2O_ISTA_TASK_LASSO 1
typedef struct {
  int32_t form;            /* L2O_ISTA_LISTA, _COUPLED, _LFISTA or _LAMP */
  int32_t batch, m, n;     /* > 0 */
  int32_t num_layers;      /* K: sizes theta, step, ss_rank and the W slots */
  int32_t k0, k1;          /* layers run: 0 <= k0 < k1 <= K */
  int32_t share_W;         /* 0 or 1 */
  const float* A;          /* [M][N] (coupled form) */
  const float* B1;         /* [N][M] (LISTA form) */
  const float* W;          /* W slots (see above) */
  const float* theta;      /* [K] */
  const float* step;       /* [K] s_k, or NULL: every s_k = 1 */
  const int32_t* ss_rank;  /* [K] support-selection ranks (>= N reads as N-1, < 0 as soft shrinkage), or NULL: soft
                              shrinkage in every layer */
  const float* y;          /* [B] rows of stride ldy >= M */
  int64_t ldy;
  const float* x_in;       /* [B][N] x_{k0}, or NULL: zeros */
  float* xs;               /* [k1-k0][B][N] out: x_{k0+1} .. x_{k1} */
  float* zs;               /* [k1-k0][B][N] out: z_k before shrinkage, or NULL (required by the backward) */
  float* rs;               /* [k1-k0][B][M] out: coupled r_k = y - x_k A^T, or NULL (required by the backward) */
  uint8_t* sel;            /* [k1-k0][B][N] out: 1 where support selection passed z through, or NULL (required by the
                              backward with ss_rank) */
  const float* W2;         /* LFISTA: Wm slots [N][N], slot k-1 for layer k (slot 0 is never read) */
  const float* s2_in;      /* the second state at k0: LFISTA x_{k0-1} [B][N], LAMP v_{k0-1} [B][M]; NULL: zeros */
  float* rowrec;           /* LAMP: [k1-k0][B][2] out: sqrt(rvar_k) and b_k of each row, or NULL (required by the
                              backward) */
} l2o_ista_args;
typedef struct {
  const float* d_xk;       /* [B][N] dL/dx_{k1} */
  float* d_x_in;           /* optional [B][N] out: dL/dx_{k0} */
  double* dW;              /* W slots out, or NULL: W is a constant (ALISTA) */
  double* dB1;             /* [N][M] out (LISTA form, required) */
  double* dtheta;          /* [K] out */
  double* dstep;           /* [K] out, or NULL */
  const float* gscale;     /* [K] gradient multipliers by creation layer, or NULL: all 1 */
  void* scratch;           /* l2o_ista_workspace_bytes */
  double* dW2;             /* LFISTA: Wm slots out, or NULL */
  const float* d_s2;       /* optional: dL/dx_{k1-1} (LFISTA) or dL/dv_{k1-1} (LAMP) from beyond the pass */
  float* d_s2_in;          /* optional out: dL/dx_{k0-1} (LFISTA) or dL/dv_{k0-1} (LAMP) */
} l2o_ista_grads;
typedef struct {
  int32_t task;            /* L2O_ISTA_TASK_SC: 0.5 ||x - x_true||^2;  LASSO: 0.5 (0.5 ||x A^T - y||^2) + lam ||x||_1 */
  int32_t batch, m, n;
  const float* A;          /* [M][N] (lasso) */
  const float* y;          /* rows of stride ldy (lasso) */
  int64_t ldy;
  const float* x_true;     /* rows of stride ldx (sc) */
  int64_t ldx;
  const float* x;          /* [B][N] x_K */
  float lam;
  float* d_x;              /* [B][N] out: dL/dx_K */
  double* loss;            /* optional [B] out: the loss of each row */
} l2o_ista_loss_args;
int l2o_ista_workspace_bytes(const l2o_ista_args* a, size_t* bytes);
int l2o_ista_fwd(const l2o_ista_args* a, void* stream);
int l2o_ista_bwd(const l2o_ista_args* a, const l2o_ista_grads* g, void* stream);
int l2o_ista_loss_grad(const l2o_ista_loss_args* a, void* stream);

/* ---------------------------------------------------------------------------------------------------------------
 * L2O-Minimax's Twin-L2O (MM = Model_Free_L2O/L2O-Minimax/Twin-L2O.py): two coordinate-wise optimizers, net 0 (min)
 * and net 1 (max), each LSTMCell(2, H) -> LSTMCell(H, H) -> Linear(H, 1) (MM Optimizer, :676), alternating on a batch
 * of B saddle-point problems of dim coordinates; R = B dim rows, row p dim + i is coordinate i of problem p.
 *
 *   l2o_minimax_fwd   iterations [t0, t1) of do_fit (MM :152-427), one launch.  Iteration t odd: net 0 updates u
 *                     from [df/du, df/dv]; even: net 1 updates v from [df/dv, df/du], both at the current (u, v).
 *                     The active net's h and c are multiplied by rescale before its cells.  Update: t < warm_end:
 *                     x += sign(delta) lr[t-1], else x += delta out_mul.  l_t = f(u, v) after a min step, -f after
 *                     a max step.
 *   l2o_minimax_bwd   the gradient of sum_t coef[t-t0] weight[p] l_t(p) over the rows of [t0, t1) w.r.t. both nets'
 *                     parameters, each l_t reached through its own update (t >= warm_end) and every later update's
 *                     h/c chain inside [t0, t1): the states entering t0 are constants.  Two launches, deterministic.
 *   l2o_minimax_image the forward's weight image of both nets from their torch-layout parameters (one launch).
 *
 * theta of one net, l2o_minimax_theta_count(H) = 12 H^2 + 25 H + 1 floats, in state_dict order: recurs.weight_ih
 * [4H][2], recurs.weight_hh [4H][H], recurs.bias_ih [4H], recurs.bias_hh [4H], recurs2.weight_ih [4H][H],
 * recurs2.weight_hh [4H][H], recurs2.bias_ih, recurs2.bias_hh, output.weight [H], output.bias [1] (gates i, f, g, o).
 * Losses (MM ToyLoss, :612): 1 a u^2 - b v^2, 2 a u^2 - b v^2 + 2uv, 3 -b v sin(a pi u) (data [B][2] = (a, b),
 * dim = 1), 4 u^T A v (data [B][dim][dim] = A).  L2O_E_UNSUPPORTED when H > 128, dim > 32 or losses 1-3 at dim > 1.
 * Float pointers 4-byte aligned, double pointers 8-byte aligned (L2O_E_INVALID otherwise). */
#define L2O_MINIMAX_MAX_HIDDEN 128
#define L2O_MINIMAX_MAX_DIM 32
typedef struct {
  int32_t loss;            /* 1 .. 4 */
  int32_t batch, dim, hidden;
  int32_t t0, t1;          /* 1-based iterations run: 1 <= t0 < t1 */
  int32_t warm_end;        /* >= 1: iterations t < warm_end take the sign step */
  float out_mul, rescale;
  const float* lr;         /* [warm_end - 1] sign-step sizes (required when t0 < warm_end) */
  const float* theta;      /* [2][theta_count] torch-layout parameters (l2o_minimax_bwd) */
  const float* image;      /* [2][l2o_minimax_image_floats] (l2o_minimax_fwd, l2o_minimax_bwd) */
  const float* data;       /* losses 1-3: [B][2] (a, b); loss 4: [B][dim][dim] A */
  float* u;                /* [R] in/out */
  float* v;                /* [R] in/out */
  float* state;            /* [2][4][R][H] in/out: h1, c1, h2, c2 of net 0, then of net 1 */
  float* traj;             /* [t1-t0][R][2] out or NULL: u, v after each iteration */
  float* ckpt;             /* [t1-t0][R][4H+2] out or NULL: the active net's inputs, h1, c1, h2, c2 before each
                              iteration (required by the backward) */
  float* dl;               /* [t1-t0][R] out or NULL: d l_t / d x_t of the updated x (required by the backward) */
  float* lval;             /* [t1-t0][B] out or NULL: l_t of each problem */
} l2o_minimax_args;
typedef struct {
  const float* coef;       /* [t1-t0] the weight of each l_t (0 where no gradient may pass) */
  const float* weight;     /* [B] per-problem weights, or NULL: all 1 */
  double* dtheta;          /* [2][theta_count] out (overwritten) */
  void* scratch;           /* l2o_minimax_workspace_bytes */
} l2o_minimax_grads;
int64_t l2o_minimax_theta_count(int32_t hidden);
int64_t l2o_minimax_image_floats(int32_t hidden);
int l2o_minimax_image(const float* theta, float* image, int32_t hidden, void* stream);
int l2o_minimax_workspace_bytes(const l2o_minimax_args* a, size_t* bytes);
int l2o_minimax_fwd(const l2o_minimax_args* a, void* stream);
int l2o_minimax_bwd(const l2o_minimax_args* a, const l2o_minimax_grads* g, void* stream);

/* ---------------------------------------------------------------------------------------------------------------
 * The analytic families of L2O-Scale's problem zoo (SC/problems/problem_generator.py, SC/ =
 * Model_Free_L2O/L2O-Scale/L2O-Scale-Training/): the objective and its gradient, or its Hessian times a vector, at
 * one parameter vector x of n coordinates, in ONE launch.  Sums are fp64 in a fixed order (no atomics): the same
 * input gives the same bits, eager or replayed from a CUDA graph.
 *
 *   l2o_zoo_value_grad  f(x) (fp64 sums, fp32 out) and out = df/dx    objective + tf.gradients (Problem.gradients, :329-350)
 *   l2o_zoo_hvp         out = H(x) v, closed forms per family          tf.gradients(grads, params, grad_ys=v)
 *
 * Families (x flattened in the reference's parameter order):
 *   QUADRATIC  0.5 ||A x - y||^2, A [n][n]            LASSO  QUADRATIC + p0 ||x||_1
 *   BOWL       0.5 ||A x||^2, A [2][2] (y NULL)        NORM   (sum_i (|A x - y|_i + 1e-6)^p0)^(1/p0)
 *   RASTRIGIN  mean_i(0.5 (A x - y)_i^2) - p0 c.cos(2 pi x) + p0 n^2   (y = b)
 *   PROJECTION_QUADRATIC  sum_bi (x_i A_bi)^2           SUM_OF_QUADRATICS  sum_bi (x_i - A_bi)^2 - A_bi^2 + 1e-12
 *   OUTWARD_SNAKE  sum_b A_b0 / (|x| + 1e-6) + sum_b,i>=1 ((x_i - pi cos x_(i-1)) A_bi)^2
 *                  (A = the data batch [rows][n]: the three data families)
 *   ISOTROPIC_QUADRATIC sum x^2   DEPENDENCY_CHAIN (n = ndim + 1)   MIN_MAX_WELL   and the 2-D test functions
 *   ROSENBROCK .. MICHALEWICZ (n = 2).
 * Matrix and data families with rows * n >= 65536 run on one cluster of 8 CTAs, each owning a block of A's rows (a
 * row-block GEMV), the partial column sums exchanged through distributed shared memory and summed in rank order;
 * every other problem runs on one CTA.  L2O_E_INVALID: NULL x / out (or v for l2o_zoo_hvp, A for the matrix and data
 * families, y for QUADRATIC / LASSO / NORM / RASTRIGIN, c for RASTRIGIN), an unknown family, n or rows out of
 * range for the family (matrix families: rows == n; BOWL and the 2-D functions: n == 2; DEPENDENCY_CHAIN,
 * OUTWARD_SNAKE: n >= 2), NORM with p0 <= 0.  L2O_E_UNSUPPORTED: n > L2O_ZOO_MAX_N.
 * The non-smooth points follow TensorFlow's gradients: sign(0) = 0 for |.|, sqrt'(0) = inf (Ackley at the origin,
 * OUTWARD_SNAKE at x = 0 give NaN), ties of min / max share the gradient evenly.
 * NORM at a residual r_i = 0 exactly: d sign / dr = 0, so row i adds no curvature (its H v and Hessian-form weight is 0).
 * RASTRIGIN at a residual r_i = 0 exactly: tf.norm's r / |r| is NaN, so every entry of df/dx, H v, q and dq/dx is NaN. */
#define L2O_ZOO_MAX_N 4096
#define L2O_ZOO_QUADRATIC 0
#define L2O_ZOO_LASSO 1
#define L2O_ZOO_RASTRIGIN 2
#define L2O_ZOO_BOWL 3
#define L2O_ZOO_NORM 4
#define L2O_ZOO_PROJECTION_QUADRATIC 5
#define L2O_ZOO_SUM_OF_QUADRATICS 6
#define L2O_ZOO_OUTWARD_SNAKE 7
#define L2O_ZOO_ISOTROPIC_QUADRATIC 8
#define L2O_ZOO_DEPENDENCY_CHAIN 9
#define L2O_ZOO_MIN_MAX_WELL 10
#define L2O_ZOO_ROSENBROCK 11
#define L2O_ZOO_SADDLE 12
#define L2O_ZOO_LOGSUMEXP 13
#define L2O_ZOO_ACKLEY 14
#define L2O_ZOO_BEALE 15
#define L2O_ZOO_BOOTH 16
#define L2O_ZOO_STYBLINSKI_TANG 17
#define L2O_ZOO_MATYAS 18
#define L2O_ZOO_BRANIN 19
#define L2O_ZOO_MICHALEWICZ 20
#define L2O_ZOO_NUM_FAMILIES 21
typedef struct {
  int32_t family;          /* L2O_ZOO_* */
  int32_t n;               /* coordinates */
  int32_t rows;            /* rows of A (matrix families: n, BOWL: 2; data families: the batch); else ignored */
  float p0;                /* LASSO lambda, RASTRIGIN alpha, NORM power */
  const float* x;          /* [n] */
  const float* v;          /* [n] the direction (l2o_zoo_hvp) */
  const float* A;          /* [rows][n] row-major: the matrix (W, BOWL's sqrt(H) R) or the data batch */
  const float* y;          /* [rows] */
  const float* c;          /* [n] RASTRIGIN's c */
  float* f;                /* [1] out or NULL (l2o_zoo_value_grad) */
  float* out;              /* [n] out: df/dx (l2o_zoo_value_grad) or H v (l2o_zoo_hvp) */
} l2o_zoo_args;
int l2o_zoo_value_grad(const l2o_zoo_args* a, void* stream);
int l2o_zoo_hvp(const l2o_zoo_args* a, void* stream);

/* The Hessian form of k direction pairs (u_k, v_k) in ONE launch, closed forms per family:
 *   q   = sum_k u_k^T H(x) v_k                 (fp64 sums, fp32 out; q may be NULL)
 *   out = dq/dx = sum_k d3f(x)[u_k, v_k, .]    (exactly 0 for the families with a constant Hessian: QUADRATIC, LASSO,
 *                                               BOWL, ISOTROPIC_QUADRATIC, PROJECTION_QUADRATIC, SUM_OF_QUADRATICS,
 *                                               BOOTH, MATYAS, SADDLE)
 * With U = V = Rademacher probes, q / k is Hutchinson's estimate of tr H and out / k its gradient; with k = 1 out is
 * the x-adjoint of l2o_zoo_hvp (u = the adjoint of H v, v = the direction).  base carries the problem as for
 * l2o_zoo_hvp (its v and f are not read; out receives dq/dx).  Same launch rule, argument rules and non-smooth
 * conventions as l2o_zoo_hvp; in addition L2O_E_INVALID: NULL U, V or out, or k < 1; L2O_E_UNSUPPORTED:
 * k > L2O_ZOO_MAX_PAIRS (q and out are sums over pairs: split k into chunks and add). */
#define L2O_ZOO_MAX_PAIRS 10
typedef struct {
  l2o_zoo_args base;       /* the problem, x and out */
  int32_t k;               /* direction pairs, 1 .. L2O_ZOO_MAX_PAIRS */
  const float* U;          /* [k][n] */
  const float* V;          /* [k][n]; may be U */
  float* q;                /* [1] out or NULL */
} l2o_zoo_form_args;
int l2o_zoo_hess_form(const l2o_zoo_form_args* a, void* stream);

/* Number of this library's kernels launched so far in this process (bench.py's gpu_launches). */
int64_t l2o_launch_count(void);
const char* l2o_status_string(int status);
const char* l2o_last_cuda_error(void);
const char* l2o_version(void);

#ifdef __cplusplus
}
#endif
#endif /* L2O_B200_H_ */
