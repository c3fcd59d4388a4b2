/* gm_b200 — C ABI of the H100-native GAN/VAE train-step hot path.
 *
 * The reference (shayneobrien/generative-models) is pure Python/PyTorch and has no
 * FFI of its own; each entry point below replaces the reference call sites cited
 * beside it (paths relative to the reference tree).  Conventions:
 *   - every function returns 0 on success, a negative GM_ERR_* otherwise;
 *     gm_last_error(ctx) holds a message.  Nothing throws across the ABI.
 *   - all pointers named *_dev are DEVICE pointers; work is ENQUEUED on the
 *     caller's cudaStream_t (passed as void*), never synchronised.
 *   - the caller (torch) owns parameter / gradient / optimizer-state storage; the
 *     library borrows the pointers given to gm_gan_bind until re-bind/destroy and
 *     owns only its workspaces and bf16 operand copies.
 *   - one engine per process per GPU; not re-entrant on one engine from 2 threads.
 */
#ifndef GM_B200_H_
#define GM_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define GM_OK 0
#define GM_ERR_ARG (-1)
#define GM_ERR_CUDA (-2)
#define GM_ERR_STATE (-3)
#define GM_ERR_UNSUPPORTED (-4)

typedef struct gm_ctx gm_ctx;
typedef struct gm_gan gm_gan;
typedef struct gm_vae gm_vae;
typedef void* gm_stream; /* cudaStream_t */

/* loss variants: one per reference file (SURVEY.md A.1) */
typedef enum {
  GM_NS = 0,      /* src/ns_gan.py:172-216      */
  GM_MM,          /* src/mm_gan.py:195-237      */
  GM_W,           /* src/w_gan.py:190-229       */
  GM_WGP,         /* src/w_gp_gan.py:177-239    */
  GM_LS,          /* src/ls_gan.py:173-215      */
  GM_DRA,         /* src/dra_gan.py:174-245     */
  GM_RA,          /* src/ra_gan.py:183-229      */
  GM_FISHER,      /* src/fisher_gan.py:193-248  */
  GM_F_TV, GM_F_FKL, GM_F_RKL, GM_F_PEARSON, GM_F_HELLINGER, GM_F_JS, /* src/f_gan.py:99-142 */
  GM_INFO,        /* src/info_gan.py:223-304    */
  GM_BEGAN        /* src/be_gan.py:212-258 (D is an autoencoder, flat layout [encoder.W|.b|decoder.W|.b]) */
} gm_variant;

typedef enum { GM_OUT_SIGMOID = 0, GM_OUT_RELU = 1, GM_OUT_NONE = 2 } gm_out_act;
typedef enum { GM_IMG_F32 = 0, GM_IMG_U8 = 1, GM_IMG_BITS = 2 } gm_img_fmt;
typedef enum { GM_NET_G = 0, GM_NET_D = 1 } gm_net;
/* arithmetic of the tensor-core GEMM operands (SURVEY.md 8b dtype_mode):
 *   GM_PREC_BF16  : bf16 operands (8-bit mantissa), fp32 accumulation — the speed mode (BASELINE configs[1..3]);
 *   GM_PREC_SPLIT : every operand is carried as a bf16 pair hi + lo (16-bit mantissa) and each product runs as
 *                   three tensor-core passes hi*hi + hi*lo + lo*hi into the same fp32 accumulator: fp32-grade
 *                   gradients (north_star's 1e-3 bound against the reference's fp32 CPU autograd) at ~1/3 speed. */
typedef enum { GM_PREC_BF16 = 0, GM_PREC_SPLIT = 1 } gm_prec;

/* torch.optim.Adam hyper-parameters (src/ns_gan.py:107-110, src/vae.py:139-142);
 * clamp > 0 applies WGAN weight clipping after the update (src/w_gan.py:158). */
typedef struct {
  float lr, beta1, beta2, eps, weight_decay, clamp;
} gm_adam_hp;

int gm_version(void);
int gm_ctx_create(int device, gm_ctx** out);
int gm_ctx_destroy(gm_ctx* ctx);
const char* gm_last_error(const gm_ctx* ctx);
int gm_ctx_num_sms(const gm_ctx* ctx);

/* ---- dense building blocks (unit tests; level-(ii) interception) ------------
 * C[M,N] = epilogue( sum_k A(m,k) B(n,k) ), bf16 operands, fp32 accumulate, on
 * wgmma tensor cores.  Replaces ATen addmm/mm under nn.Linear
 * (src/ns_gan.py:44-45,58-59) and autograd's AddmmBackward (src/ns_gan.py:138,155).
 *   mode 0 "NT": A_dev [M, lda] (K contiguous), B_dev [N, ldb] (K contiguous)
 *   mode 1 "TN": A_dev [K, lda] (M contiguous), B_dev [K, ldb] (N contiguous);
 *                (contraction over batch rows: dW = X^T dY; any K)
 * out_kind 0: bf16 C_dev [M, ldc] with optional bias[N], act (0 none, 1 relu,
 *             2 sigmoid, 3 LeakyReLU(act_slope)), aux (bf16 [M, ld_aux];
 *             aux_mode 1: *= aux(1-aux), 2: *= (aux > 0), 3: v = sigmoid
 *             output, aux = target x: stores -2 (x - v) v (1 - v) and adds
 *             sum (x - v)^2 over the row's columns < N to its dot_out slots);
 *             columns [N, out_cols) are written as padding (col N = 1 if
 *             pad_one).  dot_w/dot_out: optional fused row-dot of the stored
 *             values; dot_out holds 2*ceil(out_cols/BN) partial slots of dot_ld
 *             floats (BN = 64 if out_cols <= 64, else 208) whose sum is the row's
 *             value.  Rows >= M and columns [out_cols, ldc) are not written.
 * out_kind 1: fp32 C_dev (ldc floats; transposed store if transpose), split-K
 *             partials summed by the library into C_dev.  Only the logical
 *             block ([M, N], or [N, M] transposed) is written.
 * Refused with GM_ERR_ARG before any launch: mode outside 0..1; mode 1 with a
 * bf16 output; act outside 0..3 or aux_mode outside 0..3; aux_mode without
 * aux_dev or the reverse; an fp32 output with any epilogue field (out_cols
 * other than 0 or N, pad_one, bias, act, aux, dot_w, dot_out); transpose on a
 * bf16 output; a bf16 output with N % 16, out_cols % 8, ldc % 8 or ld_aux % 8
 * not 0, ldc < out_cols or ld_aux < out_cols; an fp32 ldc below the stored
 * row length (N, or M transposed); C_dev, aux_dev, bias_dev or dot_w_dev not
 * 16-byte aligned; dot_w_dev without dot_out_dev; dot_ld < M. */
typedef struct {
  int mode, M, N, K;
  const void* A_dev; int lda;
  const void* B_dev; int ldb;
  int out_kind;
  void* C_dev; int ldc;
  int out_cols, pad_one;
  const float* bias_dev; int act;
  const void* aux_dev; int ld_aux, aux_mode;
  const float* dot_w_dev; float* dot_out_dev; int dot_ld;
  int transpose;
  float act_slope;   /* act 3 = LeakyReLU(act_slope) */
} gm_gemm_desc;
int gm_gemm_bf16(gm_ctx* ctx, const gm_gemm_desc* d, gm_stream stream);

/* One fused Adam update over n contiguous fp32 elements; `step` is the 1-based
 * step count (bias correction).  Replaces optim.Adam.step (src/ns_gan.py:139,156). */
int gm_adam_step(gm_ctx* ctx, float* p_dev, const float* g_dev, float* m_dev, float* v_dev, int n,
                 const gm_adam_hp* hp, int step, gm_stream stream);
/* gm_adam_step with the learning rate hp->lr * lr_scale_dev[0] (a device scalar, e.g. BEGAN's plateau scheduler, read at
 * run time); lr_scale_dev NULL is gm_adam_step. */
int gm_adam_step_lr(gm_ctx* ctx, float* p_dev, const float* g_dev, float* m_dev, float* v_dev, int n,
                    const gm_adam_hp* hp, const float* lr_scale_dev, int step, gm_stream stream);

/* ---- GAN train-step engine --------------------------------------------------
 * MLP generator z -> hidden -> image (sigmoid) and discriminator image -> hidden
 * -> 1 (src/ns_gan.py:35-60).  Flat fp32 parameter layout per net, in
 * nn.Module.parameters() order: [linear.weight | linear.bias | out.weight | out.bias]. */
typedef struct {
  int image_size, hidden_dim, z_dim; /* NSGAN(image_size, hidden_dim, z_dim), src/ns_gan.py:66 */
  int max_batch;                     /* largest local batch */
  int variant;                       /* gm_variant */
  int d_out_act;                     /* gm_out_act: sigmoid, or relu for src/w_gp_gan.py:61 */
  int dtype_mode;                    /* gm_prec */
} gm_gan_desc;

int gm_gan_create(gm_ctx* ctx, const gm_gan_desc* desc, gm_gan** out);
int gm_gan_destroy(gm_gan* gan);
int gm_gan_param_count(const gm_gan* gan, int net);
int gm_gan_bind(gm_gan* gan, int net, float* params_dev, float* grads_dev, float* exp_avg_dev, float* exp_avg_sq_dev);
/* refresh the bf16 operand copies from the bound fp32 parameters (after init /
 * load_state_dict, src/ns_gan.py:287-290) */
int gm_gan_sync_shadows(gm_gan* gan, int net, gm_stream stream);

/* train_D + D_loss.backward() (src/ns_gan.py:172-194,138): forward G (fresh noise),
 * D on real and fake rows, variant loss, backward through D only; writes the flat D
 * gradient (already scaled by inv_global_batch so data-parallel ranks SUM) and the
 * loss (loss_dev[0]).  noise_dev [batch, z] fp32 or NULL for on-device Philox
 * (seed, step); aux_dev: WGAN-GP eps [batch] / DRAGAN (delta [batch] then u
 * [batch, image_size]) or NULL for on-device Philox; gather_idx_dev: optional row
 * indices into images_dev (the DataLoader shuffle of src/ns_gan.py:222-226). */
int gm_gan_d_grad(gm_gan* gan, const void* images_dev, int img_fmt, const int* gather_idx_dev, int batch,
                  const float* noise_dev, const float* aux_dev, float inv_global_batch, uint64_t seed,
                  uint64_t step, float* loss_dev, gm_stream stream);
/* process_batch of the next train_D ahead of time (stages the real rows; the following gm_gan_d_grad with the same batch
 * skips its staging).  `step` = the step the later gm_gan_d_grad is called with. */
int gm_gan_d_stage(gm_gan* gan, const void* images_dev, int img_fmt, const int* gather_idx_dev, int batch, uint64_t step, gm_stream stream);
/* train_G + G_loss.backward() (src/ns_gan.py:196-216,155), G gradients only. */
int gm_gan_g_grad(gm_gan* gan, int batch, const float* noise_dev, float inv_global_batch, uint64_t seed,
                  uint64_t step, float* loss_dev, gm_stream stream);
/* gm_gan_g_grad in two halves: the generator forward G(z) of train_G (src/ns_gan.py:207-208) does not depend
 * on the D update that precedes it, so a data-parallel host may enqueue it while the D-gradient exchange
 * (gm_gan_apply_allreduce on another stream) is still in flight, then wait for that stream and run the rest. */
int gm_gan_g_forward_stage(gm_gan* gan, int batch, const float* noise_dev, uint64_t seed, uint64_t step, gm_stream stream);
int gm_gan_g_grad_staged(gm_gan* gan, int batch, float inv_global_batch, float* loss_dev, gm_stream stream);
/* optimizer.step() on one net (src/ns_gan.py:139,156) + operand-copy refresh. */
int gm_gan_apply(gm_gan* gan, int net, const gm_adam_hp* hp, int step, gm_stream stream);
/* Lazy gradients (single-GPU fast path): with on != 0, *_grad leaves the gradient as split-K
 * partials and the following gm_gan_apply(net) gathers, stores the flat gradient AND applies
 * Adam in one kernel (one launch and one pass over the partials less per update).  The flat
 * gradient buffer is then valid only after gm_gan_apply; call gm_gan_materialize_grads to
 * form it earlier (e.g. before an all-reduce).  Any later *_grad call materialises pending
 * gradients first, so results never depend on the mode. */
int gm_gan_set_lazy_grads(gm_gan* gan, int on, gm_stream stream);
int gm_gan_materialize_grads(gm_gan* gan, gm_stream stream);
/* ---- data-parallel optimizer step: gradient all-reduce fused into Adam --------
 * The only exchange of the path is the SUM of the flat D / G gradient (one process per GPU).
 * gm_comm owns a peer-mapped exchange buffer: create one per process, exchange the 64-byte
 * gm_comm_handle of every rank (the host uses torch.distributed for that), gm_comm_open them.
 * gm_gan_apply_allreduce then replaces `all_reduce(grad); optimizer.step()` (src/ns_gan.py:139,156
 * under data parallelism) by ONE kernel per rank that publishes its gradient chunk by chunk,
 * sums the peers' chunks over NVLink in rank order and applies Adam.  Collective: every rank
 * calls it with the same net and step, in the same order. */
typedef struct gm_comm gm_comm;
int gm_comm_create(gm_ctx* ctx, int nfloats, gm_comm** out);
int gm_comm_handle(gm_comm* comm, void* out64);
int gm_comm_open(gm_comm* comm, int rank, int world, const void* handles /* world x 64 bytes, rank order */);
int gm_comm_destroy(gm_comm* comm);
int gm_gan_apply_allreduce(gm_gan* gan, int net, const gm_adam_hp* hp, int step, gm_comm* comm, gm_stream stream);
/* The exchange in two halves: gm_gan_exchange_begin publishes this rank's gradient to every peer and never waits; the next
 * gm_gan_apply_allreduce(net) then only waits for the peers, sums and applies Adam.  Work that does not depend on the update
 * goes between them on the same stream - the generator forward of train_G (gm_gan_g_forward_stage) under the D exchange, the
 * image staging of the next train_D (gm_gan_d_stage) under the G exchange - and absorbs the NVLink latency and the ranks'
 * arrival skew. */
int gm_gan_exchange_begin(gm_gan* gan, int net, gm_comm* comm, gm_stream stream);
/* Batch statistics over the GLOBAL batch under data parallelism (RaNS mean(DG) src/ra_gan.py:204, Fisher
 * moments src/fisher_gan.py:214-218, DRAGAN images.std() src/dra_gan.py:204, BEGAN DX / DG of the K
 * controller src/be_gan.py:189-190): with a communicator attached, gm_gan_d_grad exchanges the partial
 * sums between the ranks on the device, so N ranks x B samples reproduce one process with N*B samples.
 * comm == NULL detaches (per-rank statistics). */
int gm_gan_attach_comm(gm_gan* gan, gm_comm* comm);

/* Device-step mode (CUDA-graph replay of the train step; the launch-bound small-batch regime of BASELINE configs[0]):
 * Adam's step count, the Philox streams of train_D / train_G and the sampler's round live in device counters advanced by
 * the step's own kernels, so ONE captured graph of gm_gan_d_grad, gm_gan_apply(D), gm_gan_g_grad, gm_gan_apply(G) replays
 * as successive steps of src/ns_gan.py:126-156.  counters4 = {Adam steps done on G, on D, train_G calls, train_D calls}
 * (NULL = zeros).  While on, the `step` arguments of those entry points are ignored. */
int gm_gan_use_device_step(gm_gan* gan, int on, const unsigned long long* counters4_host, gm_stream stream);
int gm_gan_device_steps(gm_gan* gan, unsigned long long* counters4_host, gm_stream stream);
/* programmatic dependent launch on / off at run time (default on; GM_NO_PDL=1 starts with it off) */
int gm_ctx_set_pdl(gm_ctx* ctx, int on);
/* Loss constants the reference passes as train_D / train_G keyword arguments (defaults = the reference's):
 * gradient-penalty LAMBDA (src/w_gp_gan.py:177), DRAGAN's K and C (src/dra_gan.py:174), LSGAN's a, b, c
 * (src/ls_gan.py:173,197).  Takes effect from the next gm_gan_d_grad / gm_gan_g_grad. */
typedef struct { float gp_lambda, gp_k, dra_c, ls_a, ls_b, ls_c; } gm_loss_consts;
int gm_gan_set_loss_consts(gm_gan* gan, const gm_loss_consts* consts);
/* On-device batch sampling — replaces `next(iter(DataLoader(shuffle=True)))` (src/ns_gan.py:222-226): with a
 * resident pool of n_pool images (images_dev of gm_gan_d_grad) and gather_idx_dev == NULL, batch row r of step
 * `step` reads pool row perm_{seed,step}(r), perm a pseudo-random permutation of [0, n_pool) drawn per step
 * (distinct rows inside a batch, like the first batch of a freshly shuffled loader).  n_pool == 0: off. */
int gm_gan_set_sampler(gm_gan* gan, long long n_pool, uint64_t seed);
/* the same permutation evaluated on the host: out_host[r] = perm_{seed,round}(offset + r), r < count */
int gm_sampler_indices_host(long long n_pool, uint64_t seed, uint64_t round, uint64_t offset, int count, int* out_host);
/* the indices that draw produces (tests, logging): idx_dev[batch] */
int gm_gan_sample_indices(gm_gan* gan, int batch, uint64_t step, int* idx_dev, gm_stream stream);
/* the N(0,1) generator noise gm_gan_d_grad (g_step 0) / gm_gan_g_grad (g_step 1) draw on the device for
 * (seed, step) when noise_dev == NULL — compute_noise of src/ns_gan.py:218-220 as in-kernel Philox —
 * as the bf16-rounded operand values, out_dev [batch, z] fp32 (tests). */
int gm_gan_debug_noise(gm_gan* gan, int batch, uint64_t seed, uint64_t step, int g_step, float* out_dev, gm_stream stream);

/* test aid: an internal bf16 activation buffer as fp32 (hi + lo planes summed in split mode) -> out_dev [rows, cols];
 * which: 0 noise operand, 1 G hidden, 2 image rows [real|fake|...], 3 D hidden, 4 D hidden gradient, 5 dL/dG-pre-sigmoid, 6 G hidden gradient */
int gm_gan_debug_read(gm_gan* gan, int which, int row0, int rows, int cols, float* out_dev, gm_stream stream);

/* D outputs of the last *_grad call (D step: batch real then batch fake; G step:
 * batch fake) -> dst_dev; what the reference names DX_score / DG_score. */
int gm_gan_scores(gm_gan* gan, float* dst_dev, int n, gm_stream stream);
/* ---- custom-loss path --------------------------------------------------------
 * README.md:31 tells users to "edit train_D and train_G": a loss written in torch on
 * DX_score / DG_score must still train.  These four calls are Generator.forward /
 * Discriminator.forward (src/ns_gan.py:43-46,57-60) and their backward halves as
 * separate entry points; the host wraps them in torch.autograd.Function objects
 * (gm_b200/gan_api.py).  `slot` in [0, gm_gan_num_slots) picks the row region that keeps
 * one D forward's activations alive until its backward.  Gradients are written to the
 * bound flat gradient buffers (overwritten per call; the host accumulates). */
int gm_gan_num_slots(const gm_gan* gan);
/* scores_dev[batch] = D(x_dev[batch, image_size]) (fp32 in, fp32 out, final activation applied) */
int gm_gan_d_forward(gm_gan* gan, int slot, const float* x_dev, int batch, float* scores_dev, gm_stream stream);
/* dscore_dev[batch] = dL/dscore -> flat D gradient; dx_dev (nullable) [batch, image_size] = dL/dx */
int gm_gan_d_backward(gm_gan* gan, int slot, int batch, const float* dscore_dev, float* dx_dev, gm_stream stream);
/* images_dev[batch, image_size] = G(noise_dev[batch, z]) keeping the activations for one backward */
int gm_gan_g_forward(gm_gan* gan, const float* noise_dev, int batch, float* images_dev, gm_stream stream);
/* dimages_dev[batch, image_size] = dL/dG(z) -> flat G gradient */
int gm_gan_g_backward(gm_gan* gan, int batch, const float* dimages_dev, gm_stream stream);

/* Generator.forward (src/ns_gan.py:43-46) for sampling: noise [n, z] fp32 -> images
 * [n, image_size] fp32. */
int gm_gan_generate(gm_gan* gan, const float* noise_dev, int n, float* images_dev, gm_stream stream);
/* InfoGAN (GM_INFO engines; generator input = z + 10 categorical + 10 continuous codes):
 * the auxiliary network Q (src/info_gan.py:78-94), flat layout [linear.W | .b | inference.W | .b];
 * g_mi_* are the G moment buffers of MI_optimizer, which spans G and Q (src/info_gan.py:146-148). */
int gm_gan_q_param_count(const gm_gan* gan);
int gm_gan_bind_q(gm_gan* gan, float* q_params_dev, float* q_grads_dev, float* q_exp_avg_dev, float* q_exp_avg_sq_dev,
                  float* g_mi_exp_avg_dev, float* g_mi_exp_avg_sq_dev);
int gm_gan_sync_shadows_q(gm_gan* gan, gm_stream stream);
/* train_Q + MI_loss.backward() (src/info_gan.py:269-304,204): CE on the categorical code
 * + MSE on the continuous code; writes the flat G and Q gradients and loss_dev[0]. */
int gm_gan_q_grad(gm_gan* gan, int batch, const float* noise_dev, int z_dim, float inv_global_batch, float* loss_dev,
                  gm_stream stream);
/* MI_optimizer.step() (src/info_gan.py:205). */
int gm_gan_apply_mi(gm_gan* gan, const gm_adam_hp* hp, int step, gm_stream stream);
/* BEGAN (GM_BEGAN engines): device state [K, scale_real, scale_fake, DX, DG, plateau best,
 * plateau bad count, lr scale, inv_b, inv_b, convergence] (src/be_gan.py:109-110,186-195);
 * gm_gan_began_control applies the proportional control of K and the ReduceLROnPlateau pair. */
int gm_gan_began_state(gm_gan* gan, float* host11, int set, gm_stream stream);
int gm_gan_began_control(gm_gan* gan, float gamma, float lambda, float patience, gm_stream stream);
/* Discriminator.forward (src/ns_gan.py:57-60) for inference: images [n, image_size]
 * (gm_img_fmt) -> scores [n] fp32. */
int gm_gan_discriminate(gm_gan* gan, const void* images_dev, int img_fmt, int n, float* scores_dev, gm_stream stream);
/* Fisher GAN scalar state (src/fisher_gan.py:117-118,155): get/set LAMBDA, RHO. */
int gm_gan_fisher_state(gm_gan* gan, float* lambda_rho_host, int set, gm_stream stream);
/* ---- VAE train-step engine (src/vae.py) ---------------------------------------
 * Encoder x -> hidden -> (mu, log_var), z = mu + eps * exp(log_var/2), Decoder z ->
 * hidden -> x (sigmoid) (src/vae.py:47-106).  Flat fp32 layout:
 * [enc.linear.W | .b | enc.mu.W | enc.log_var.W | enc.mu.b | enc.log_var.b |
 *  dec.linear.W | .b | dec.recon.W | .b]. */
typedef struct { int image_size, hidden_dim, z_dim, max_batch; int dtype_mode; /* gm_prec */ } gm_vae_desc;
int gm_vae_create(gm_ctx* ctx, const gm_vae_desc* desc, gm_vae** out);
int gm_vae_destroy(gm_vae* vae);
int gm_vae_param_count(const gm_vae* vae);
int gm_vae_bind(gm_vae* vae, float* params_dev, float* grads_dev, float* exp_avg_dev, float* exp_avg_sq_dev);
int gm_vae_sync_shadows(gm_vae* vae, gm_stream stream);
/* compute_batch + (recon + kl).backward() (src/vae.py:157-161,193-212): recon =
 * sum (x - out)^2, kl = sum 0.5 (mu^2 + exp(lv) - lv - 1); writes the flat gradient and
 * losses_dev[0..1] = {recon, kl}.  eps_dev [batch, z] fp32 or NULL for on-device Philox. */
int gm_vae_grad(gm_vae* vae, const void* images_dev, int img_fmt, const int* gather_idx_dev, int batch,
                const float* eps_dev, float grad_scale, uint64_t seed, uint64_t step, float* losses_dev,
                gm_stream stream);
/* On-device epoch shuffling for gm_vae_grad (gather_idx_dev == NULL): step s reads batch k = s mod batches_per_epoch
 * (rows [k * batch_size, k * batch_size + batch) of the permutation of epoch s / batches_per_epoch) of the resident
 * pool — the `for batch in self.train_iter` of src/vae.py:150 without host work; batch_size is the loader's nominal
 * batch (the last batch of an epoch may be shorter; 0 = the batch of the call).  n_pool == 0: off. */
int gm_vae_set_sampler(gm_vae* vae, long long n_pool, long long batches_per_epoch, long long batch_size, uint64_t seed);
/* lazy gradients, as gm_gan_set_lazy_grads: gm_vae_apply gathers the split-K partials, stores the flat gradient and
 * applies Adam in one kernel; gm_vae_materialize_grads forms the flat gradient earlier (e.g. before an all-reduce). */
int gm_vae_set_lazy_grads(gm_vae* vae, int on, gm_stream stream);
int gm_vae_materialize_grads(gm_vae* vae, gm_stream stream);
/* eps of the last gm_vae_grad / gm_vae_forward call (src/vae.py:104; the Philox draw when eps_dev was NULL) -> out_dev [batch, z] */
int gm_vae_last_eps(gm_vae* vae, float* out_dev, int batch, gm_stream stream);
/* optimizer.step() with coupled weight decay (src/vae.py:139-142,162). */
int gm_vae_apply(gm_vae* vae, const gm_adam_hp* hp, int step, gm_stream stream);
/* VAE.forward (+ losses) without gradients: evaluate / reconstruct (src/vae.py:214-252).
 * Any of out_images_dev [n, image_size], mu_logvar_dev [n, 2 z], losses_dev [2] may be NULL. */
int gm_vae_forward(gm_vae* vae, const void* images_dev, int img_fmt, int n, const float* eps_dev, uint64_t seed,
                   uint64_t step, float* out_images_dev, float* mu_logvar_dev, float* losses_dev, gm_stream stream);
/* Decoder.forward (src/vae.py:74-77) for sampling. */
int gm_vae_decode(gm_vae* vae, const float* z_dev, int n, float* out_images_dev, gm_stream stream);
/* ---- per-call encoder / decoder (a user-written compute_batch, README.md:31) -------------
 * Encoder.forward and Decoder.forward (src/vae.py:58-61,74-77) and their backward halves as separate entry points; the
 * host wraps them in torch.autograd.Function objects and composes VAE.forward from them (src/vae.py:94-106).  `slot` in
 * [0, gm_vae_num_slots) picks the buffers that keep one encoder (decoder) call's activations alive until its backward.
 * Gradients go to a caller-supplied flat gradient buffer in the engine's layout: an encoder backward writes its segments
 * [enc.linear.W .. enc.log_var.b] only, a decoder backward its segments [dec.linear.W .. dec.recon.b] only.  dz_dev
 * (nullable) [batch, z] = dL/dz.  Each call forms pending lazy gradients first.  All refuse null pointers, a slot outside
 * [0, gm_vae_num_slots) and batch outside (0, max_batch] with GM_ERR_ARG, and a split-precision engine with
 * GM_ERR_UNSUPPORTED, before anything is launched. */
int gm_vae_num_slots(const gm_vae* vae);
int gm_vae_encoder_forward(gm_vae* vae, int slot, const float* x_dev, int batch, float* mu_logvar_dev, gm_stream stream);
int gm_vae_encoder_backward(gm_vae* vae, int slot, int batch, const float* dmu_logvar_dev, float* grads_dev, gm_stream stream);
int gm_vae_decoder_forward(gm_vae* vae, int slot, const float* z_dev, int batch, float* images_dev, gm_stream stream);
int gm_vae_decoder_backward(gm_vae* vae, int slot, int batch, const float* dimages_dev, float* grads_dev, float* dz_dev,
                            gm_stream stream);
/* dL/d(pre-sigmoid output) of a sigmoid layer (the kernel of gm_vae_decoder_backward): out_rows_dev [rows, ld] bf16 holds
 * the sigmoid output out and is overwritten with dout_dev [rows, x] fp32 * out * (1 - out), 0 in columns [x, ld).
 * Refuses, with nothing launched: rows or x not positive, ld below x or not a multiple of 8, dout not 4-byte or
 * out_rows not 16-byte aligned; GM_ERR_UNSUPPORTED for 2^31 threads or more. */
int gm_sigmoid_upstream_rows(gm_ctx* ctx, const float* dout_dev, void* out_rows_dev, int rows, int x, int ld, gm_stream stream);

/* ---- conv building blocks (DCGAN path, BASELINE configs[4]; README.md:68,96 recommends DCGAN, the reference has no
 * implementation).  NHWC bf16 activations as row-major matrices [B*H*W, C]; a 4x4 stride-2 pad-1 convolution is
 * gm_im2col_k4s2 + gm_gemm_bf16, a transposed convolution gm_gemm_bf16 + gm_col2im_k4s2; their gradients are the same
 * two data movements with the roles swapped.  The DCGAN engine that sequences them is gm_b200/dcgan.py.
 * Every entry point below checks its arguments before it launches or allocates anything: GM_ERR_ARG for a NULL, non-positive,
 * out-of-range or misaligned argument, GM_ERR_UNSUPPORTED for a size the kernels' 32-bit indices cannot hold.
 * gm_im2col_k4s2: x [B*H*W, ldx] -> col [B*(H/2)*(W/2), ldc], columns (kh, kw, c).  Refused: odd H or W, ldx < C, ldc < 16 C;
 * when C is a multiple of 8 (the 16-byte path) ldx or ldc not a multiple of 8 or x / col not 16-byte aligned;
 * GM_ERR_UNSUPPORTED for 2^31 or more items (an item is 16 bytes of col, or one tap of one pixel when C % 8 != 0). */
int gm_im2col_k4s2(gm_ctx* ctx, const void* x_dev, int B, int H, int W, int C, int ldx, void* col_dev, int ldc, gm_stream stream);
/* col [B*Hi*Wi, ldc] -> y [B*2Hi*2Wi, ldy].  mode 0: sum of taps, 1: sigmoid(sum), 2: sum * LeakyReLU'(aux), 3: sum * aux (1 - aux),
 * aux [B*2Hi*2Wi, ld_aux] read in modes 2 and 3 only (aux > 0 selects slope 1; +0, -0 and negative values select `slope`).
 * Refused: mode outside 0..3, modes 2 / 3 without aux or with ld_aux < C, ldc < 16 C, ldy < C; when C is a multiple of 8 a
 * leading dimension (ld_aux in modes 2 / 3) not a multiple of 8 or col / y / aux not 16-byte aligned; GM_ERR_UNSUPPORTED for C
 * above 8 that is not a multiple of 8, and for 2^31 or more output items (pixels x C/8 groups). */
int gm_col2im_k4s2(gm_ctx* ctx, const void* col_dev, int ldc, int B, int Hi, int Wi, int C, void* y_dev, int ldy, int mode,
                   const void* aux_dev, int ld_aux, float slope, gm_stream stream);
/* nn.BatchNorm2d in training mode over NHWC rows x [rows, ld], fused with the following activation (act 0 none, 1 ReLU,
 * 2 LeakyReLU) into y [rows, ldy].  gm_bn_backward reads BOTH dy and x with leading dimension ld and writes dx [rows, lddx];
 * it expects the stats gm_bn_forward stored.  Refused by the three gm_bn_* calls: C, ld, ldy / lddx not multiples of 8, a
 * leading dimension below C, act outside 0..2, x / y / dy / dx not 16-byte aligned; GM_ERR_UNSUPPORTED for C > 2048. */
int gm_bn_forward(gm_ctx* ctx, const void* x_dev, long long rows, int C, int ld, const float* gamma_dev, const float* beta_dev, float eps,
                  int act, float slope, void* y_dev, int ldy, float* stats_dev /* [2][C]: mean, invstd */,
                  float* running_dev /* [2][C] or NULL */, float momentum, gm_stream stream);
int gm_bn_backward(gm_ctx* ctx, const void* dy_dev, const void* x_dev, long long rows, int C, int ld, const float* stats_dev,
                   const float* gamma_dev, const float* beta_dev, int act, float slope, void* dx_dev, int lddx,
                   float* dgb_dev /* [2][C]: dbeta, dgamma */, gm_stream stream);
/* fp32 [R, C] -> bf16 [R, ld] and / or its transpose [C, ld_t] (the two GEMM operand forms of a weight matrix), rounded to
 * nearest even.  Refused: both outputs NULL, ld < C with dst, ld_t < R with dst_t; GM_ERR_UNSUPPORTED for R C >= 2^31. */
int gm_cast_bf16(gm_ctx* ctx, const float* src_dev, int R, int C, void* dst_dev, int ld, void* dst_t_dev, int ld_t, gm_stream stream);
/* out [rows, ld] bf16 with column 0 = v[r], the rest 0; GM_ERR_UNSUPPORTED for rows ld >= 2^31 */
int gm_pack_col0(gm_ctx* ctx, const float* v_dev, int rows, void* out_dev, int ld, gm_stream stream);
/* process_batch (src/ns_gan.py:222-226, src/ae.py:150-151) as a standalone step: images [*, x] -> bf16 rows [rows, ld], a ones
 * column at x and zeros up to ld; row r reads image gather_idx_dev[r] (r when NULL).  GM_IMG_F32 rounds to nearest even.
 * GM_IMG_U8 and GM_IMG_BITS binarise: a u8 value becomes 1 when it is non-zero (255 and 3 alike), and the bit format is one
 * bit per value over the whole [*, x] array in np.packbits order (most significant bit first; rows are not byte aligned
 * unless x is a multiple of 8).  Refused: img_fmt outside gm_img_fmt, ld <= x or not a multiple of 8, out not 16-byte aligned,
 * fp32 images or gather_idx not 4-byte aligned. */
int gm_stage_images(gm_ctx* ctx, const void* images_dev, int img_fmt, const int* gather_idx_dev, void* out_dev, int rows, int x, int ld,
                    gm_stream stream);
/* A batch drawn from a device-resident dataset of 8-bit codes (gm_b200.dcgan.DevicePool): codes_dev [n_pool, row_vals] uint8
 * (one image per row, NHWC order, row_vals a multiple of 16, 16-byte aligned) and table_bf16_dev [256] bf16 bit patterns.
 * Batch row r reads pool row perm_{seed,round}(offset + r), the permutation of gm_sampler_indices_host, and out_bf16_dev
 * [rows, row_vals] (16-byte aligned) receives table[code] for each of its values - the NHWC bf16 rows stage_images makes of
 * that image.  idx_out_dev (nullable) receives the rows' pool indices.  GM_ERR_ARG, with nothing launched, unless
 * 0 < rows <= n_pool <= 2^31 - 1 and offset + rows <= n_pool. */
int gm_stage_pool_rows(gm_ctx* ctx, const uint8_t* codes_dev, long long n_pool, int row_vals, const uint16_t* table_bf16_dev, uint64_t seed,
                       uint64_t round, uint64_t offset, int rows, void* out_bf16_dev, int* idx_out_dev, gm_stream stream);
/* The image layout at the autograd boundary of the conv drop-ins (Generator / Discriminator forward and backward):
 * NCHW-flattened fp32 [n, ch*64*64], as the reference's process_batch flattens images (src/ns_gan.py:222-226), and the
 * kernels' NHWC bf16 rows [n*4096, ch].  gm_image_to_rows writes dst = x rounded to nearest even (tensor.to(bfloat16)),
 * or, with out_nhwc_dev (the generator's stored sigmoid output f), (x * f) * (1 - f) rounded once: the upstream of the
 * pre-sigmoid output from dL/dG(z).  gm_rows_to_image widens exactly.  GM_ERR_ARG, with nothing launched, unless n > 0,
 * 1 <= ch <= 4 and every pointer is 16-byte aligned. */
int gm_image_to_rows(gm_ctx* ctx, const float* x_nchw_dev, const void* out_nhwc_dev /* nullable */, int n, int ch, void* dst_nhwc_dev,
                     gm_stream stream);
int gm_rows_to_image(gm_ctx* ctx, const void* src_nhwc_dev, int n, int ch, float* dst_nchw_dev, gm_stream stream);
/* generator noise rows as a bf16 GEMM operand out [rows, ld]: columns [0, z) Philox N(0,1) keyed by (seed, stream_id)
 * (noise_dev NULL) or a caller tensor [rows, z] fp32 rounded to nearest even, column z = 1, zeros up to ld.  Refused: ld <= z
 * or not a multiple of 8, out not 16-byte aligned; GM_ERR_UNSUPPORTED for rows ceil((z + 1) / 8) >= 2^31. */
int gm_noise_rows(gm_ctx* ctx, const float* noise_dev, void* out_dev, int rows, int z, int ld, uint64_t seed, uint64_t stream_id,
                  gm_stream stream);
/* the adversarial loss + dL/dlogit on a logit vector (train_D: batch real then batch fake rows; train_G: batch fake rows);
 * row-wise variants only (NS, MM, W, LS, f-GAN): GM_ERR_UNSUPPORTED for the other gm_variant values, GM_ERR_ARG for a variant
 * or out_act outside their enums and for batch outside 1..2^30.  loss_dev[0] = loss, [1] = sum of ds (a fixed-order sum). */
int gm_loss_rows(gm_ctx* ctx, int variant, int out_act, const float* logits_dev, int batch, int g_step, float inv_global_batch,
                 float* ds_dev, float* d_out_dev, float* loss_dev, gm_stream stream);
/* gm_loss_rows with the loss constants of lc (the LS targets ls_a, ls_b, ls_c; the other fields are unused here); lc NULL
 * means the reference's defaults a = 0, b = 1, c = 1 (src/ls_gan.py:173,197), which is what gm_loss_rows runs. */
int gm_loss_rows_c(gm_ctx* ctx, int variant, int out_act, const float* logits_dev, int batch, int g_step, float inv_global_batch,
                   const gm_loss_consts* lc, float* ds_dev, float* d_out_dev, float* loss_dev, gm_stream stream);
/* WGAN-GP on the batch-norm-free conv critic (src/w_gp_gan.py:197-218; gm_b200/dcgan.py sequences it).
 * x_hat = eps x_real + (1 - eps) x_fake per image over NHWC rows [B*HW, C]; eps_dev [B] fp32, or NULL for Philox U(0,1]
 * keyed by (seed, stream_id); eps_out_dev [B] (nullable) receives the eps used. */
int gm_gp_interp_rows(gm_ctx* ctx, const void* xr_dev, int ldr, const void* xf_dev, int ldf, int B, int HW, int C, const float* eps_dev,
                      float* eps_out_dev, uint64_t seed, uint64_t stream_id, void* out_dev, int ldo, gm_stream stream);
/* per image b of the image gradient g [B*HW, C]: norm_dev[b] = ||g_b||, r_dev = 2 lambda inv_grad (||g_b|| - 1) / ||g_b|| g_b
 * (0 when ||g_b|| = 0) as bf16, and loss_dev[0] += lambda inv_loss sum_b (||g_b|| - 1)^2 (loss_dev nullable) */
int gm_gp_penalty(gm_ctx* ctx, const void* g_dev, int ldg, int B, int HW, int C, float lambda, float inv_grad, float inv_loss,
                  void* r_dev, int ldr, float* norm_dev, float* loss_dev, gm_stream stream);
/* gm_im2col_k4s2 of x * LeakyReLU'(m) (m > 0 selects slope 1, anything else `slope`), the product rounded once.  Refused like
 * gm_im2col_k4s2, and: C, ldx, ldm or ldc not a multiple of 8, ldm < C, x / m / col not 16-byte aligned. */
int gm_im2col_k4s2_lrelu_mask(gm_ctx* ctx, const void* x_dev, int B, int H, int W, int C, int ldx, const void* m_dev, int ldm, float slope,
                              void* col_dev, int ldc, gm_stream stream);
/* out = x * LeakyReLU'(m) over rows [rows, C]; out may alias x or m.  Refused: C or a leading dimension not a multiple of 8 or
 * below C, x / m / out not 16-byte aligned; GM_ERR_UNSUPPORTED for rows C / 8 >= 2^31. */
int gm_lrelu_mask_rows(gm_ctx* ctx, const void* x_dev, int ldx, const void* m_dev, int ldm, long long rows, int C, float slope,
                       void* out_dev, int ldo, gm_stream stream);
/* Batch-statistic D losses (RaNS src/ra_gan.py:204-205, Fisher src/fisher_gan.py:214-223) on a logit vector [real B | fake B],
 * split so that data-parallel ranks can SUM the statistics between the calls.  bstat = the global batch the statistics run
 * over (B x ranks).  stats: 8 doubles, [0..3] = phase 0 (sum d real, sum d fake, sum d^2 real, sum d^2 fake), [4] = phase 1
 * (RaNS: sum over the real rows of q(1-q)/(q+1e-8), q = sigmoid(d - mean d_fake), given the global phase-0 sums in
 * stats_in_dev).  gm_loss_rows_stats then writes ds_dev[2B] = dL/dlogit (scaled by inv_global_batch), d_out_dev (nullable),
 * loss_dev[0] = loss (local means, global statistics), [1] = sum ds, [2] = Fisher's Omega, and for Fisher updates
 * fisher_state_dev[0] (lambda) by -rho Omega with fisher_state_dev[1] = rho (src/fisher_gan.py:155). */
int gm_loss_stats(gm_ctx* ctx, int variant, int out_act, const float* logits_dev, int batch, long long bstat, int phase,
                  const double* stats_in_dev, double* stats_out_dev, gm_stream stream);
int gm_loss_rows_stats(gm_ctx* ctx, int variant, int out_act, const float* logits_dev, int batch, float inv_global_batch,
                       const double* stats_dev, long long bstat, float* fisher_state_dev, float* ds_dev, float* d_out_dev,
                       float* loss_dev, gm_stream stream);
/* DRAGAN (src/dra_gan.py:200-219) on contiguous image rows [rows, cols] (cols a multiple of 8, 16-byte aligned).
 * gm_dra_std_sums: sums_dev[2] = (sum x, sum x^2) of this process's rows.  gm_dra_xhat_rows: with the global sums and their
 * element count, x_hat = delta x + (1 - delta)(x + C std(x) u) (std unbiased); rnd_dev = [delta (rows) | u (rows x cols, the
 * rows' own element order)] or NULL for Philox keyed by (seed, stream_id).  gm_dra_penalty: per x_hat image b with logit
 * s_b and J_b = d s_b / d image: norm_dev[b] = ||g_b|| = sigma'(s_b) ||J_b||, the tangent seed
 * r_b = k sigma' [J_b/||J_b|| + (1 - 2 sigma) ||J_b|| x_hat_b], k = 2 lambda inv_grad (||g_b|| - K) (0 when ||J_b|| = 0), and
 * loss_dev[0] += lambda inv_loss sum_b (||g_b|| - K)^2 (loss_dev nullable). */
int gm_dra_std_sums(gm_ctx* ctx, const void* x_dev, int rows, int cols, int ld, double* sums_dev, gm_stream stream);
int gm_dra_xhat_rows(gm_ctx* ctx, const void* x_dev, int rows, int cols, int ld, const double* sums_dev, double count, float dra_c,
                     const float* rnd_dev, uint64_t seed, uint64_t stream_id, void* out_dev, int ldo, gm_stream stream);
int gm_dra_penalty(gm_ctx* ctx, const void* J_dev, int ldj, const void* xhat_dev, int ldx, const float* logits_dev, int B, int HW, int C,
                   float lambda, float K, float inv_grad, float inv_loss, void* r_dev, int ldr, float* norm_dev, float* loss_dev,
                   gm_stream stream);
/* BEGAN (src/be_gan.py:212-258) on the conv autoencoder D; images are contiguous rows [rows, cols] (cols a multiple of 8,
 * 16-byte aligned).  gm_l1_rows: grad_dev = sign(r - x) inv (coef_dev ? coef_dev[0] : 1) as bf16 (sign(0) = 0) and
 * sum_dev[0] = sum |r - x| (one double, a fixed-order reduction, for data-parallel ranks to SUM).  gm_began_loss_final: from
 * the summed doubles over `batch` (the global batch) images, D step: loss_dev[0] = DX - K DG, state [3], [4] = DX, DG; G step
 * (g_step != 0, sum_x_dev unused): loss_dev[0] = DG.  gm_began_control: K and the ReduceLROnPlateau pair on a caller-owned
 * state_dev[11] (the layout of gm_gan_began_state).  gm_began_dfake_rows: out = (T - dr) f (1 - f), the G step's
 * dL/d(pre-sigmoid G output) from T = D's input gradient at f = G(z) and dr = gm_l1_rows' grad. */
int gm_l1_rows(gm_ctx* ctx, const void* r_dev, const void* x_dev, int rows, int cols, float inv, const float* coef_dev, void* grad_dev,
               double* sum_dev, gm_stream stream);
int gm_began_loss_final(gm_ctx* ctx, const double* sum_x_dev, const double* sum_g_dev, int batch, int g_step, float* state_dev,
                        float* loss_dev, gm_stream stream);
int gm_began_control(gm_ctx* ctx, float* state_dev, float gamma, float lambda, float patience, gm_stream stream);
int gm_began_dfake_rows(gm_ctx* ctx, const void* T_dev, const void* dr_dev, const void* fake_dev, void* out_dev, int rows, int cols,
                        gm_stream stream);
/* InfoGAN (src/info_gan.py:269-325) on the conv path.  gm_info_noise_rows: compute_noise on the device, Philox keyed by
 * (seed, stream_id): out_dev [rows, ld] bf16 = [z (zd) N(0,1) | one-hot of a category uniform over [0, nd) | nc N(0,1) | 1 | 0
 * ...] (the layout of gm_noise_rows' rows, ld a multiple of 8, > zd + nd + nc) and codes_dev [rows, zd + nd + nc] fp32 = the
 * same values (every one bf16-representable).  gm_info_loss_rows: on Q's rows q_dev [rows, ldq] fp32 ([0, nd) categorical
 * logits, [nd, nd + nc) continuous code) and the codes [rows, ldc] (one-hot at [zd, zd + nd), continuous at [zd + nd, zd + nd
 * + nc)): loss_dev[0] = mean CE + mean squared error over rows x nc, grad_dev [rows, ldo] bf16 = (softmax - onehot) inv and
 * 2 (q - c) inv / nc (inv = inv_global_batch), zero in columns [nd + nc, ldo). */
int gm_info_noise_rows(gm_ctx* ctx, void* out_dev, int ld, float* codes_dev, int rows, int zd, int nd, int nc, uint64_t seed,
                       uint64_t stream_id, gm_stream stream);
int gm_info_loss_rows(gm_ctx* ctx, const float* q_dev, int ldq, const float* codes_dev, int ldc, int zd, int rows, int nd, int nc,
                      float inv_global_batch, void* grad_dev, int ldo, float* loss_dev, gm_stream stream);
/* The VAE (src/vae.py:94-106,193-212) on the conv path.  gm_sse_sigmoid_rows: on contiguous rows [rows, cols] (cols a multiple
 * of 8, 16-byte aligned) of the decoder's sigmoid output out_dev and the target x_dev (bf16): sum_dev[0] = sum (x - out)^2
 * (one double, a fixed-order reduction, for data-parallel ranks to SUM) and grad_dev = 2 scale (out - x) out (1 - out) as
 * bf16, dL/d(pre-sigmoid output).  gm_vae_latent_rows: on the encoder head's fp32 rows mulv_dev [rows, ldm] ([0, z) mu,
 * [z, 2z) log_var), z = mu + eps e^(lv/2) with eps from eps_in_dev [rows, z] or Philox keyed by (seed, stream_id) (stream_id
 * below 2^58), eps_out_dev [rows, z] = the eps used, zrows_dev [rows, ldz] bf16 = [z | 1 | 0 ...] (ldz a multiple of 8 above
 * z), kl_sum_dev[0] = sum 0.5 (mu^2 + e^lv - lv - 1) (one double, fixed order).  gm_vae_dlatent_rows: from dz_dev [rows,
 * lddz] fp32 = dL/dz, out_dev [rows, ld] bf16 = scale [mu + dz | 0.5 (e^lv - 1) + 0.5 dz eps e^(lv/2) | 0 ...], the upstream
 * of the encoder head.  gm_bn_forward_eval: nn.BatchNorm2d in inference mode over NHWC rows, fused with the activation like
 * gm_bn_forward, with the running statistics running_dev [2][C] (mean, var), which it does not update. */
int gm_sse_sigmoid_rows(gm_ctx* ctx, const void* out_dev, const void* x_dev, int rows, int cols, float scale, void* grad_dev,
                        double* sum_dev, gm_stream stream);
int gm_vae_latent_rows(gm_ctx* ctx, const float* mulv_dev, int ldm, const float* eps_in_dev, float* eps_out_dev, void* zrows_dev, int ldz,
                       int rows, int z, uint64_t seed, uint64_t stream_id, double* kl_sum_dev, gm_stream stream);
int gm_vae_dlatent_rows(gm_ctx* ctx, const float* mulv_dev, int ldm, const float* dz_dev, int lddz, const float* eps_dev, void* out_dev,
                        int ld, int rows, int z, float scale, gm_stream stream);
int gm_bn_forward_eval(gm_ctx* ctx, const void* x_dev, long long rows, int C, int ld, const float* gamma_dev, const float* beta_dev,
                       const float* running_dev, float eps, int act, float slope, void* y_dev, int ldy, gm_stream stream);
/* The autoencoder (src/ae.py:38-39,147-160) on the conv path: the code is relu of the encoder head's linear output.
 * gm_ae_latent_rows: on the head's fp32 rows h_dev [rows, ldm], zrows_dev [rows, ldz] bf16 = [relu(h) | 1 | 0 ...] (the
 * decoder's input rows, the layout of gm_vae_latent_rows).  gm_ae_dlatent_rows: from dz_dev [rows, lddz] fp32 = dL/dcode,
 * out_dev [rows, ld] bf16 = [dz 1[h > 0] | 0 ...] (0 at h == 0, as torch's relu backward), the upstream of the head.  Both
 * refuse, with nothing launched: rows or z not positive, ldm / lddz below z, ldz not above z or ld below z, ldz / ld not a
 * multiple of 8, h / dz not 4-byte or zrows / out not 16-byte aligned; GM_ERR_UNSUPPORTED for 2^31 threads or more. */
int gm_ae_latent_rows(gm_ctx* ctx, const float* h_dev, int ldm, void* zrows_dev, int ldz, int rows, int z, gm_stream stream);
int gm_ae_dlatent_rows(gm_ctx* ctx, const float* h_dev, int ldm, const float* dz_dev, int lddz, void* out_dev, int ld, int rows, int z,
                       gm_stream stream);

/* number of this library's kernels launched since the last call with reset != 0 */
long long gm_launch_count(gm_ctx* ctx, int reset);
/* measurement aid (bench.py roofline): record CUDA events around every tensor-core
 * GEMM launch on its launch stream; gm_prof_collect synchronises and returns, per
 * kernel instantiation (4 slots), total ms, algorithmic FLOPs and launch count. */
int gm_prof_enable(gm_ctx* ctx, int on);   /* 0 off, 1 GEMM launches by kind (gm_prof_collect), 2 every launch by name (gm_prof_report) */
/* level-2 report: synchronises and writes "name,launches,total_ms" lines (in first-launch order) into buf; returns bytes needed */
int gm_prof_report(gm_ctx* ctx, char* buf, int buflen);
int gm_prof_collect(gm_ctx* ctx, double* ms4, double* flops4, long long* count4);

#ifdef __cplusplus
}
#endif
#endif /* GM_B200_H_ */
