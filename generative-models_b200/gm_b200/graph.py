"""CUDA-graph replay of the fused train step (the launch-bound small-batch regime: BASELINE configs[0] runs the
reference at batch 64, src/ns_gan.py:311-314; its default is 100, src/utils.py:16).

One train step = ~22 kernel launches of a few microseconds each at these sizes, so the step is bound by launch
latency, not by the GPU.  `GraphedGanStep` captures ONE step (gm_gan_d_grad, gm_gan_apply(D), gm_gan_g_grad,
gm_gan_apply(G)) into a CUDA graph with the engine in device-step mode (Adam step counts, Philox streams and the
batch sampler's round live in device counters the kernels advance themselves) and replays it: every replay is the
next train step of src/ns_gan.py:126-156, with one launch from the host."""
import torch

from . import _lib
from ._lib import GmError


class GraphedGanStep:
    """step = GraphedGanStep(eng, pool_bits, n_pool, batch, hpD, hpG, seed); step() runs one train step; step.losses
    is the engine's [D_loss, G_loss] device buffer.  Requires the resident bit-packed pool + on-device noise (nothing
    in the step may depend on host data)."""

    def __init__(self, eng, pool_bits, n_pool, batch, hpD, hpG, seed=0, inv_global_batch=None, warmup=3):
        self.eng, self.batch = eng, batch
        self.pool, self.n_pool, self.hpD, self.hpG, self.seed = pool_bits, n_pool, hpD, hpG, int(seed)
        self.inv = inv_global_batch
        eng.set_lazy_grads(True)
        eng.set_sampler(n_pool, seed)
        eng.use_device_step(True)
        for _ in range(max(warmup, 1)):          # shapes, plans and kernel attributes are set up outside the capture
            self._one()
        torch.cuda.synchronize()
        self.graph = torch.cuda.CUDAGraph()
        self.pdl = True
        try:
            with torch.cuda.graph(self.graph):
                self._one()
        except RuntimeError:
            # a driver that rejects programmatic-dependent-launch edges in a capture: plain edges instead
            _lib.check(eng.h, _lib.lib().gm_ctx_set_pdl(eng.h, 0))
            self.pdl = False
            torch.cuda.synchronize()
            self.graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(self.graph):
                self._one()
        self.losses = eng.loss_buf

    def _one(self):
        eng, B = self.eng, self.batch
        eng.d_grad(self.pool, fmt="bits", batch=B, inv_global_batch=self.inv, seed=self.seed)
        eng.apply(1, self.hpD)
        eng.g_grad(B, inv_global_batch=self.inv, seed=self.seed)
        eng.apply(0, self.hpG)

    def __call__(self):
        self.graph.replay()

    def close(self):
        """Back to host-driven steps (reads the device counters back into the engine)."""
        torch.cuda.synchronize()
        self.eng.use_device_step(False)
        if not self.pdl:
            _lib.check(self.eng.h, _lib.lib().gm_ctx_set_pdl(self.eng.h, 1))


def graphed_gan_step(workload, steps):
    """bench.py small-batch leg: time `steps` graph replays of an NSGAN bench.Workload -> {value, ms_per_step}."""
    eng = workload.eng
    step = GraphedGanStep(eng, workload.bits, workload.N, workload.B, workload.hpD, workload.hpG, workload.seed, workload.inv)
    for _ in range(10):
        step()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        step()
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1)
    losses = [float(v) for v in step.losses.tolist()]
    ctr = eng.device_steps()
    step.close()
    return {"value": round(workload.B * steps / (ms * 1e-3), 1), "ms_per_step": round(ms / steps, 4), "pdl_edges": step.pdl,
            "losses_last_step": losses, "device_counters": ctr}
