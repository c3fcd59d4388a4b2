"""ctypes binding of libgm_b200.so (C ABI: include/gm_b200.h)."""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
# GM_B200_LIB: load an alternative build of the same library (kernel A/B experiments, tools/)
lib_path = os.environ.get("GM_B200_LIB") or os.path.join(_HERE, "lib", "libgm_b200.so")


class GmError(RuntimeError):
    pass


VARIANTS = {"ns": 0, "mm": 1, "w": 2, "wgp": 3, "ls": 4, "dra": 5, "ra": 6, "fisher": 7,
            "f_total_variation": 8, "f_forward_kl": 9, "f_reverse_kl": 10, "f_pearson": 11,
            "f_hellinger": 12, "f_jensen_shannon": 13, "info": 14, "began": 15}
OUT_ACTS = {"sigmoid": 0, "relu": 1, "none": 2}
IMG_FMTS = {"f32": 0, "u8": 1, "bits": 2}
PRECISIONS = {"bf16": 0, "split": 1}      # include/gm_b200.h: gm_prec


class AdamHP(C.Structure):
    _fields_ = [("lr", C.c_float), ("beta1", C.c_float), ("beta2", C.c_float), ("eps", C.c_float),
                ("weight_decay", C.c_float), ("clamp", C.c_float)]

    @classmethod
    def make(cls, lr, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0, clamp=0.0):
        return cls(lr, betas[0], betas[1], eps, weight_decay, clamp)


class GemmDesc(C.Structure):
    _fields_ = [("mode", C.c_int), ("M", C.c_int), ("N", C.c_int), ("K", C.c_int),
                ("A", C.c_void_p), ("lda", C.c_int), ("B", C.c_void_p), ("ldb", C.c_int),
                ("out_kind", C.c_int), ("Cp", C.c_void_p), ("ldc", C.c_int),
                ("out_cols", C.c_int), ("pad_one", C.c_int),
                ("bias", C.c_void_p), ("act", C.c_int),
                ("aux", C.c_void_p), ("ld_aux", C.c_int), ("aux_mode", C.c_int),
                ("dot_w", C.c_void_p), ("dot_out", C.c_void_p), ("dot_ld", C.c_int),
                ("transpose", C.c_int), ("act_slope", C.c_float)]


class LossConsts(C.Structure):
    _fields_ = [("gp_lambda", C.c_float), ("gp_k", C.c_float), ("dra_c", C.c_float), ("ls_a", C.c_float), ("ls_b", C.c_float),
                ("ls_c", C.c_float)]


class VaeDesc(C.Structure):
    _fields_ = [("image_size", C.c_int), ("hidden_dim", C.c_int), ("z_dim", C.c_int), ("max_batch", C.c_int),
                ("dtype_mode", C.c_int)]


class SghmcHP(C.Structure):
    """include/gm_b200.h: gm_sghmc_hp (gm_bgan_apply)"""
    _fields_ = [("lr", C.c_float), ("alpha", C.c_float), ("prior_std", C.c_float), ("data_size", C.c_float)]


class GanDesc(C.Structure):
    _fields_ = [("image_size", C.c_int), ("hidden_dim", C.c_int), ("z_dim", C.c_int),
                ("max_batch", C.c_int), ("variant", C.c_int), ("d_out_act", C.c_int), ("dtype_mode", C.c_int)]


_lib = None


def lib():
    """Load libgm_b200.so; fail loudly if it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(lib_path):
        raise GmError("libgm_b200.so is not built (%s). Run `python -c 'import __graft_entry__ as g; g.build()'` "
                      "at the repo root. There is no CPU / eager fallback." % lib_path)
    L = C.CDLL(lib_path)
    vp, i, f, u64 = C.c_void_p, C.c_int, C.c_float, C.c_uint64
    L.gm_version.restype = i
    L.gm_ctx_create.argtypes = [i, C.POINTER(vp)]
    L.gm_ctx_destroy.argtypes = [vp]
    L.gm_last_error.argtypes = [vp]
    L.gm_last_error.restype = C.c_char_p
    L.gm_ctx_num_sms.argtypes = [vp]
    L.gm_launch_count.argtypes = [vp, i]
    L.gm_launch_count.restype = C.c_longlong
    L.gm_prof_enable.argtypes = [vp, i]
    L.gm_prof_report.argtypes = [vp, C.c_char_p, i]
    L.gm_prof_collect.argtypes = [vp, C.POINTER(C.c_double), C.POINTER(C.c_double), C.POINTER(C.c_longlong)]
    L.gm_gemm_bf16.argtypes = [vp, C.POINTER(GemmDesc), vp]
    L.gm_adam_step.argtypes = [vp, vp, vp, vp, vp, i, C.POINTER(AdamHP), i, vp]
    L.gm_adam_step_lr.argtypes = [vp, vp, vp, vp, vp, i, C.POINTER(AdamHP), vp, i, vp]
    L.gm_gan_create.argtypes = [vp, C.POINTER(GanDesc), C.POINTER(vp)]
    L.gm_gan_destroy.argtypes = [vp]
    L.gm_gan_param_count.argtypes = [vp, i]
    L.gm_gan_bind.argtypes = [vp, i, vp, vp, vp, vp]
    L.gm_gan_sync_shadows.argtypes = [vp, i, vp]
    L.gm_gan_d_grad.argtypes = [vp, vp, i, vp, i, vp, vp, f, u64, u64, vp, vp]
    L.gm_gan_d_stage.argtypes = [vp, vp, i, vp, i, u64, vp]
    L.gm_gan_g_grad.argtypes = [vp, i, vp, f, u64, u64, vp, vp]
    L.gm_gan_g_forward_stage.argtypes = [vp, i, vp, u64, u64, vp]
    L.gm_gan_g_grad_staged.argtypes = [vp, i, f, vp, vp]
    L.gm_gan_apply.argtypes = [vp, i, C.POINTER(AdamHP), i, vp]
    L.gm_gan_scores.argtypes = [vp, vp, i, vp]
    L.gm_gan_generate.argtypes = [vp, vp, i, vp, vp]
    L.gm_gan_q_param_count.argtypes = [vp]
    L.gm_gan_bind_q.argtypes = [vp, vp, vp, vp, vp, vp, vp]
    L.gm_gan_sync_shadows_q.argtypes = [vp, vp]
    L.gm_gan_q_grad.argtypes = [vp, i, vp, i, f, vp, vp]
    L.gm_gan_apply_mi.argtypes = [vp, C.POINTER(AdamHP), i, vp]
    L.gm_gan_began_state.argtypes = [vp, C.POINTER(C.c_float), i, vp]
    L.gm_gan_began_control.argtypes = [vp, f, f, f, vp]
    L.gm_gan_discriminate.argtypes = [vp, vp, i, i, vp, vp]
    L.gm_gan_num_slots.argtypes = [vp]
    L.gm_comm_create.argtypes = [vp, i, C.POINTER(vp)]
    L.gm_comm_handle.argtypes = [vp, vp]
    L.gm_comm_open.argtypes = [vp, i, i, vp]
    L.gm_comm_destroy.argtypes = [vp]
    L.gm_gan_attach_comm.argtypes = [vp, vp]
    L.gm_gan_exchange_begin.argtypes = [vp, i, vp, vp]
    L.gm_gan_apply_allreduce.argtypes = [vp, i, C.POINTER(AdamHP), i, vp, vp]
    L.gm_gan_set_lazy_grads.argtypes = [vp, i, vp]
    L.gm_gan_materialize_grads.argtypes = [vp, vp]
    L.gm_gan_d_forward.argtypes = [vp, i, vp, i, vp, vp]
    L.gm_gan_d_backward.argtypes = [vp, i, i, vp, vp, vp]
    L.gm_gan_g_forward.argtypes = [vp, vp, i, vp, vp]
    L.gm_gan_g_backward.argtypes = [vp, i, vp, vp]
    L.gm_gan_ae_forward.argtypes = [vp, i, vp, i, vp, vp]
    L.gm_gan_ae_backward.argtypes = [vp, i, i, vp, vp, vp]
    L.gm_gan_num_q_slots.argtypes = [vp]
    L.gm_gan_q_forward.argtypes = [vp, i, vp, i, vp, vp]
    L.gm_gan_q_backward.argtypes = [vp, i, i, vp, vp, vp]
    L.gm_vae_create.argtypes = [vp, C.POINTER(VaeDesc), C.POINTER(vp)]
    L.gm_vae_destroy.argtypes = [vp]
    L.gm_vae_param_count.argtypes = [vp]
    L.gm_vae_bind.argtypes = [vp, vp, vp, vp, vp]
    L.gm_vae_sync_shadows.argtypes = [vp, vp]
    L.gm_vae_grad.argtypes = [vp, vp, i, vp, i, vp, f, u64, u64, vp, vp]
    L.gm_vae_apply.argtypes = [vp, C.POINTER(AdamHP), i, vp]
    L.gm_vae_forward.argtypes = [vp, vp, i, i, vp, u64, u64, vp, vp, vp, vp]
    L.gm_vae_decode.argtypes = [vp, vp, i, vp, vp]
    L.gm_vae_num_slots.argtypes = [vp]
    L.gm_vae_encoder_forward.argtypes = [vp, i, vp, i, vp, vp]
    L.gm_vae_encoder_backward.argtypes = [vp, i, i, vp, vp, vp]
    L.gm_vae_decoder_forward.argtypes = [vp, i, vp, i, vp, vp]
    L.gm_vae_decoder_backward.argtypes = [vp, i, i, vp, vp, vp, vp]
    L.gm_sigmoid_upstream_rows.argtypes = [vp, vp, vp, i, i, i, vp]
    ll = C.c_longlong
    L.gm_im2col_k4s2.argtypes = [vp, vp, i, i, i, i, i, vp, i, vp]
    L.gm_col2im_k4s2.argtypes = [vp, vp, i, i, i, i, i, vp, i, i, vp, i, f, vp]
    L.gm_bn_forward.argtypes = [vp, vp, ll, i, i, vp, vp, f, i, f, vp, i, vp, vp, f, vp]
    L.gm_bn_backward.argtypes = [vp, vp, vp, ll, i, i, vp, vp, vp, i, f, vp, i, vp, vp]
    L.gm_cast_bf16.argtypes = [vp, vp, i, i, vp, i, vp, i, vp]
    L.gm_pack_col0.argtypes = [vp, vp, i, vp, i, vp]
    L.gm_stage_images.argtypes = [vp, vp, i, vp, vp, i, i, i, vp]
    L.gm_stage_pool_rows.argtypes = [vp, vp, ll, i, vp, u64, u64, u64, i, vp, vp, vp]
    L.gm_image_to_rows.argtypes = [vp, vp, vp, i, i, vp, vp]
    L.gm_rows_to_image.argtypes = [vp, vp, i, i, vp, vp]
    L.gm_noise_rows.argtypes = [vp, vp, vp, i, i, i, u64, u64, vp]
    L.gm_loss_rows.argtypes = [vp, i, i, vp, i, i, f, vp, vp, vp, vp]
    L.gm_loss_rows_c.argtypes = [vp, i, i, vp, i, i, f, C.POINTER(LossConsts), vp, vp, vp, vp]
    L.gm_gp_interp_rows.argtypes = [vp, vp, i, vp, i, i, i, i, vp, vp, u64, u64, vp, i, vp]
    L.gm_gp_penalty.argtypes = [vp, vp, i, i, i, i, f, f, f, vp, i, vp, vp, vp]
    L.gm_im2col_k4s2_lrelu_mask.argtypes = [vp, vp, i, i, i, i, i, vp, i, f, vp, i, vp]
    L.gm_lrelu_mask_rows.argtypes = [vp, vp, i, vp, i, ll, i, f, vp, i, vp]
    L.gm_loss_stats.argtypes = [vp, i, i, vp, i, ll, i, vp, vp, vp]
    L.gm_loss_rows_stats.argtypes = [vp, i, i, vp, i, f, vp, ll, vp, vp, vp, vp, vp]
    L.gm_dra_std_sums.argtypes = [vp, vp, i, i, i, vp, vp]
    L.gm_dra_xhat_rows.argtypes = [vp, vp, i, i, i, vp, C.c_double, f, vp, u64, u64, vp, i, vp]
    L.gm_dra_penalty.argtypes = [vp, vp, i, vp, i, vp, i, i, i, f, f, f, f, vp, i, vp, vp, vp]
    L.gm_l1_rows.argtypes = [vp, vp, vp, i, i, f, vp, vp, vp, vp]
    L.gm_began_loss_final.argtypes = [vp, vp, vp, i, i, vp, vp, vp]
    L.gm_began_control.argtypes = [vp, vp, f, f, f, vp]
    L.gm_began_dfake_rows.argtypes = [vp, vp, vp, vp, vp, i, i, vp]
    L.gm_info_noise_rows.argtypes = [vp, vp, i, vp, i, i, i, i, u64, u64, vp]
    L.gm_info_loss_rows.argtypes = [vp, vp, i, vp, i, i, i, i, i, f, vp, i, vp, vp]
    L.gm_sse_sigmoid_rows.argtypes = [vp, vp, vp, i, i, f, vp, vp, vp]
    L.gm_vae_latent_rows.argtypes = [vp, vp, i, vp, vp, vp, i, i, i, u64, u64, vp, vp]
    L.gm_vae_dlatent_rows.argtypes = [vp, vp, i, vp, i, vp, vp, i, i, i, f, vp]
    L.gm_bn_forward_eval.argtypes = [vp, vp, ll, i, i, vp, vp, vp, f, i, f, vp, i, vp]
    L.gm_ae_latent_rows.argtypes = [vp, vp, i, vp, i, i, i, vp]
    L.gm_ae_dlatent_rows.argtypes = [vp, vp, i, vp, i, vp, i, i, i, vp]
    L.gm_gan_use_device_step.argtypes = [vp, i, vp, vp]
    L.gm_gan_device_steps.argtypes = [vp, vp, vp]
    L.gm_ctx_set_pdl.argtypes = [vp, i]
    L.gm_gan_set_loss_consts.argtypes = [vp, C.POINTER(LossConsts)]
    L.gm_gan_set_sampler.argtypes = [vp, C.c_longlong, u64]
    L.gm_sampler_indices_host.argtypes = [C.c_longlong, u64, u64, u64, i, vp]
    L.gm_gan_sample_indices.argtypes = [vp, i, u64, vp, vp]
    L.gm_gan_debug_read.argtypes = [vp, i, i, i, i, vp, vp]
    L.gm_gan_debug_noise.argtypes = [vp, i, u64, u64, i, vp, vp]
    L.gm_vae_set_lazy_grads.argtypes = [vp, i, vp]
    L.gm_vae_materialize_grads.argtypes = [vp, vp]
    L.gm_vae_last_eps.argtypes = [vp, vp, i, vp]
    L.gm_vae_debug_read.argtypes = [vp, i, i, i, i, vp, vp]
    L.gm_vae_set_sampler.argtypes = [vp, C.c_longlong, C.c_longlong, C.c_longlong, u64]
    L.gm_gan_fisher_state.argtypes = [vp, C.POINTER(C.c_float), i, vp]
    L.gm_bir_vae_create.argtypes = [vp, C.POINTER(VaeDesc), f, C.POINTER(vp)]
    L.gm_bir_vae_grad.argtypes = [vp, vp, i, vp, i, vp, vp, f, u64, u64, vp, vp]
    L.gm_bir_vae_forward.argtypes = [vp, vp, i, i, vp, vp, f, u64, u64, vp, vp, vp, vp]
    L.gm_bir_vae_last_latent.argtypes = [vp, vp, vp, i, vp]
    L.gm_mmd_gaussian.argtypes = [vp, vp, vp, i, i, f, vp, vp, vp]
    L.gm_cvae_create.argtypes = [vp, C.POINTER(VaeDesc), i, C.POINTER(vp)]
    L.gm_cvae_grad.argtypes = [vp, vp, i, vp, vp, i, vp, u64, u64, vp, vp]
    L.gm_cvae_forward.argtypes = [vp, vp, i, vp, i, vp, u64, u64, vp, vp, vp, vp]
    L.gm_cvae_decode.argtypes = [vp, vp, vp, i, vp, vp]
    L.gm_cvae_encoder_forward.argtypes = [vp, i, vp, vp, i, vp, vp]
    L.gm_cvae_decoder_forward.argtypes = [vp, i, vp, vp, i, vp, vp]
    L.gm_aae_create.argtypes = [vp, C.POINTER(VaeDesc), C.POINTER(vp)]
    L.gm_aae_d_param_count.argtypes = [vp]
    L.gm_aae_bind_d.argtypes = [vp, vp, vp, vp, vp, vp, vp]
    L.gm_aae_sync_shadows_d.argtypes = [vp, vp]
    L.gm_aae_recon_grad.argtypes = [vp, vp, i, vp, i, u64, vp, vp]
    L.gm_aae_d_grad.argtypes = [vp, i, vp, u64, u64, vp, vp]
    L.gm_aae_g_grad.argtypes = [vp, i, vp, vp]
    L.gm_aae_apply_d.argtypes = [vp, C.POINTER(AdamHP), i, vp]
    L.gm_aae_apply_g.argtypes = [vp, C.POINTER(AdamHP), i, vp]
    L.gm_aae_forward.argtypes = [vp, vp, i, i, vp, vp, vp, vp]
    L.gm_aae_last_prior.argtypes = [vp, vp, i, vp]
    L.gm_aae_num_d_slots.argtypes = [vp]
    L.gm_aae_d_forward.argtypes = [vp, i, vp, i, vp, vp]
    L.gm_aae_d_backward.argtypes = [vp, i, i, vp, vp, vp]
    L.gm_bgan_create.argtypes = [vp, C.POINTER(GanDesc), i, C.POINTER(vp)]
    L.gm_bgan_num_samples.argtypes = [vp]
    L.gm_bgan_g_stride.argtypes = [vp]
    L.gm_bgan_d_grad.argtypes = [vp, vp, i, vp, i, vp, u64, u64, vp, vp]
    L.gm_bgan_g_grad.argtypes = [vp, i, vp, u64, u64, vp, vp]
    L.gm_bgan_apply.argtypes = [vp, i, C.POINTER(SghmcHP), u64, u64, vp]
    L.gm_bgan_generate.argtypes = [vp, i, vp, i, vp, vp]
    L.gm_bgan_sghmc_noise.argtypes = [vp, i, u64, u64, vp, vp]
    _lib = L
    return L


_ctx = {}


def ctx(device=None):
    """Per-device context handle (created on first use). Raises without an H100."""
    import torch
    if device is None:
        device = torch.cuda.current_device() if torch.cuda.is_available() else 0
    if device in _ctx:
        return _ctx[device]
    L = lib()
    h = C.c_void_p()
    rc = L.gm_ctx_create(int(device), C.byref(h))
    if rc != 0:
        msg = L.gm_last_error(h).decode() if h else "gm_ctx_create failed"
        raise GmError("gm_b200: %s (rc=%d)" % (msg, rc))
    _ctx[device] = h
    return h


def check(h, rc):
    if rc != 0:
        raise GmError("gm_b200: %s (rc=%d)" % (lib().gm_last_error(h).decode(), rc))


def _stream():
    import torch
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


def launch_count(reset=False):
    return int(lib().gm_launch_count(ctx(), 1 if reset else 0))


GEMM_KINDS = ["gemm_wgmma<208,K-major>", "gemm_wgmma<64,K-major>", "gemm_wgmma<256,MN-major>",
              "gemm_wgmma<64,MN-major>"]


def prof_enable(on=True):
    """True / 1: events around GEMM launches by kind (prof_collect); 2: around every launch by name (prof_report)."""
    check(ctx(), lib().gm_prof_enable(ctx(), int(on)))


def prof_report():
    """-> list of (kernel name, launches, total ms) in first-launch order (after prof_enable(2))."""
    buf = C.create_string_buffer(1 << 16)
    n = lib().gm_prof_report(ctx(), buf, len(buf))
    if n < 0:
        check(ctx(), n)
    out = []
    for line in buf.value.decode().splitlines():
        name, cnt, ms = line.rsplit(",", 2)
        out.append((name, int(cnt), float(ms)))
    return out


def prof_collect():
    """-> list of (kernel name, total ms, algorithmic flops, launches)."""
    ms, fl, cn = (C.c_double * 4)(), (C.c_double * 4)(), (C.c_longlong * 4)()
    check(ctx(), lib().gm_prof_collect(ctx(), ms, fl, cn))
    return [(GEMM_KINDS[k], ms[k], fl[k], cn[k]) for k in range(4)]


def gemm_bf16(A, B, out, mode="nt", N=None, K=None, M=None, bias=None, act=0, aux=None, aux_mode=0, pad_one=False,
              out_cols=None, dot_w=None, dot_out=None, transpose=False, act_slope=0.2):
    """Thin wrapper over gm_gemm_bf16 for torch CUDA tensors (unit tests, level-(ii)
    use).  mode 'nt': A [M, lda] / B [N, ldb] bf16 with K contiguous;  mode 'tn':
    A [K, lda] / B [K, ldb] bf16 (contraction over rows).  `out` bf16 [M, ldc] or fp32."""
    import torch
    d = GemmDesc()
    d.mode = 0 if mode == "nt" else 1
    if mode == "nt":
        d.M = M if M is not None else A.shape[0]
        d.N = N if N is not None else B.shape[0]
        d.K = K if K is not None else A.shape[1]
    else:
        d.K = K if K is not None else A.shape[0]
        d.M = M if M is not None else A.shape[1]
        d.N = N if N is not None else B.shape[1]
    d.A, d.lda, d.B, d.ldb = A.data_ptr(), A.stride(0), B.data_ptr(), B.stride(0)
    d.out_kind = 1 if out.dtype == torch.float32 else 0
    d.Cp, d.ldc = out.data_ptr(), out.stride(0)
    d.out_cols = out_cols if out_cols is not None else d.N
    d.pad_one = int(pad_one)
    d.bias = bias.data_ptr() if bias is not None else None
    d.act = act
    d.aux = aux.data_ptr() if aux is not None else None
    d.ld_aux = aux.stride(0) if aux is not None else 0
    d.aux_mode = aux_mode
    d.dot_w = dot_w.data_ptr() if dot_w is not None else None
    d.dot_out = dot_out.data_ptr() if dot_out is not None else None
    d.dot_ld = dot_out.stride(0) if dot_out is not None else 0
    d.transpose = int(transpose)
    d.act_slope = act_slope
    h = ctx()
    check(h, lib().gm_gemm_bf16(h, C.byref(d), _stream()))


def adam_step(p, g, m, v, hp, step, lr_scale=None):
    """One Adam update; lr_scale: None or a device fp32 scalar tensor multiplying hp.lr when the kernel runs"""
    h = ctx()
    check(h, lib().gm_adam_step_lr(h, _ptr(p), _ptr(g), _ptr(m), _ptr(v), p.numel(), C.byref(hp), _ptr(lr_scale), int(step), _stream()))
