"""gm_b200 — host-side binding of libgm_b200.so (the H100-native GAN/VAE train-step
engine).  PyTorch is used for device memory, streams and torch.distributed only;
all hot-path compute runs in the hand-written sm_90a kernels behind the C ABI
declared in include/gm_b200.h.  There is no CPU or eager-PyTorch fallback: importing
works anywhere, but creating a context without an H100 raises."""
from ._lib import (GmError, lib, lib_path, ctx, gemm_bf16, adam_step, launch_count,  # noqa: F401
                   VARIANTS, OUT_ACTS, IMG_FMTS, PRECISIONS, AdamHP, prof_enable, prof_collect, prof_report)
from .engine import GanEngine, InfoGanEngine, VaeEngine  # noqa: F401

HAS_SPLIT_PRECISION = True       # fp32-grade split-bf16 operand mode (gm_prec GM_PREC_SPLIT)
from .graph import GraphedGanStep, graphed_gan_step  # noqa: E402,F401
from .dcgan import DcganEngine, DevicePool  # noqa: E402,F401
from .ae import AeEngine  # noqa: E402,F401
