"""Elementwise conformance of every route gm_gemm_bf16 can take, against float64 (GPU).

Each case computes ref = A B^T (+ bias) in float64 from the same bf16 operands and bounds every output element:
  accumulation  e = C_ACC * ceil(K / 16) * 2^-23 * S,   S = |A| |B|^T (+ |bias|)   (about one fp32 rounding per 16-deep step)
  fp32 output   |got - ref| <= e
  bf16 output   |got - f(ref)| <= 2^-8 (|f(ref)| + m) + m,   m = L_f e + e_f + 2^-20 |f(ref)|
where 2^-8 is the unit roundoff of bf16 (8 significant bits: round-to-nearest moves a value by up to 2^-8 of itself), f is
the epilogue (activation, then the aux factor), L_f its Lipschitz constant, e_f the stated error of the
tanh.approx sigmoid and 2^-20 |f(ref)| a few fp32 roundings of the epilogue's own arithmetic.  The row-dot and SSE slots
are bounded the same way (their fp32 sum adds N 2^-24 of the summed magnitudes).  Besides the bounds, the cases check
what the kernels must leave alone bit for bit (rows >= M, columns past out_cols or past the fp32 row, dot slots of rows
>= M), the exact padding columns, exact zeros of the ReLU mask, NaN in every operand byte the kernels must not read, the
plan kind each case was meant to reach, and identities between routes that share one mainloop.  With GM_PARITY_DIR set,
the worst error-to-bound ratio of each case group is written to $GM_PARITY_DIR/parity_gemm_conformance.json."""
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import dcgan_harness as H

pytestmark = pytest.mark.gpu
_REPORT = H.Report("gemm_conformance")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

C_ACC = 4                          # accumulation bound: C_ACC fp32 roundings of S per 16-deep MMA step
E_TANH = 2.0 ** -11                # absolute error of tanh.approx.f32
E_SIG = E_TANH / 2 + 2.0 ** -24    # sigmoid = 0.5 tanh(x / 2) + 0.5, and its final fma
E_OPS = 2.0 ** -20                 # relative: the few fp32 roundings of the epilogue arithmetic
U_BF16 = 2.0 ** -8                 # unit roundoff of bf16
PAT16 = 0x4B4B                     # prefill of bf16 outputs (a finite bf16, ~1.3e7)
PAT32 = 0x4B4B4B4B                 # prefill of fp32 outputs and dot slots
KINDS = {"nt208": 0, "nt64": 1, "tn256": 2, "tn64": 3}

# bf16 epilogues: bias, act, aux_mode, row-dot, pad_one, dot_out (aux 3's SSE)
EPIS = {
    "plain": dict(),
    "bias_relu": dict(bias=True, act=1),
    "bias_sigmoid": dict(bias=True, act=2),
    "bias_relu_dot_padone": dict(bias=True, act=1, dot=True, pad_one=True),
    "aux1": dict(aux=1),
    "aux2": dict(aux=2),
    "bias_sigmoid_aux3": dict(bias=True, act=2, aux=3, sse=True),
    "lrelu": dict(act=3),
    "bias_lrelu": dict(bias=True, act=3),
    "bias": dict(bias=True),
    "relu": dict(act=1),
    "sigmoid": dict(act=2),
    "bias_aux1": dict(bias=True, aux=1),
    "relu_aux2": dict(act=1, aux=2),
    "dot": dict(dot=True),
}
# (M, N, K, out_cols - N) per tile; epilogue i takes shape i % 8, so every M, N and K of the selection meets several epilogues.
# K = 56 and 120 end on a k-block of 56 (the only ragged blocks whose last 16-deep step holds data), K = 65 on one of 1,
# M = 1 / 15 / 17 / 129 leave the 16-row epilogue slices partly empty, 128 x 300 runs several tiles per CTA, and N = 416
# with out_cols 432 adds a third n-tile that holds nothing but padding.
SHAPES = {"nt64": [(1005, 48, 784, 16), (1, 16, 8, 0), (15, 64, 56, 0), (17, 48, 65, 16),
                   (128, 16, 120, 8), (129, 64, 48, 0), (128 * 300, 64, 64, 0), (128, 48, 4096, 8)],
          "nt208": [(1005, 400, 784, 16), (17, 80, 16, 0), (128, 208, 56, 0), (129, 416, 65, 16),
                    (1, 256, 120, 8), (15, 624, 48, 0), (128 * 300, 224, 64, 0), (1005, 128, 4096, 8)]}


def _bf16_case(name, tile):
    i = list(EPIS).index(name)
    M, N, K, extra = SHAPES[tile][i % 8]
    e = EPIS[name]
    if e.get("pad_one") and extra == 0:
        extra = 16
    oc = N + extra
    return dict(name="%s_%s" % (name, tile), mode="nt", M=M, N=N, K=K, out="bf16", out_cols=oc, ldc=oc + 8 * (i % 2),
                lda=(K + 7) // 8 * 8 + 8, ldb=(K + 7) // 8 * 8 + 8, bias=e.get("bias", False), act=e.get("act", 0), slope=0.2,
                aux=e.get("aux", 0), dot=e.get("dot", False), sse=e.get("sse", False), pad_one=e.get("pad_one", False),
                transpose=False, tile=tile, group="bf16_" + name, seed=100 + i)


BF16_CASES = [_bf16_case(n, t) for t in ("nt208", "nt64") for n in EPIS]

# fp32: (mode, M, N, K, transpose, ldc, split-K).  Split-K follows from the tile count: one split when the tiles alone fill
# the SMs (or K is one k-block), up to 64 splits otherwise.  ldc 30, 38, 74, 2, 1005 and 129-wide transposed rows do not
# start on 16 bytes.
F32 = [("nt", 64, 30, 4096, False, 30, True), ("nt", 1005, 30, 784, False, 38, True), ("nt", 17, 2, 8, False, 2, False),
       ("nt", 128 * 300, 74, 64, False, 74, False), ("nt", 129, 100, 784, True, 136, True), ("nt", 30, 48, 120, True, 30, True),
       ("nt", 1005, 400, 64, False, 448, False),
       ("tn", 400, 30, 4096, False, 30, True), ("tn", 64, 20, 64, False, 64, False), ("tn", 785, 400, 8192, True, 832, True),
       ("tn", 2, 74, 256, False, 74, True), ("tn", 784, 401, 128, False, 404, True), ("tn", 4096, 2048, 256, False, 2048, False),
       ("tn", 1005, 30, 1005, True, 1005, True)]


def _f32_case(i, mode, M, N, K, tr, ldc, split):
    r8 = lambda v: (v + 7) // 8 * 8 + 8
    lda, ldb = (r8(K), r8(K)) if mode == "nt" else (r8(M), r8(N))
    tile = (("nt64" if N <= 64 else "nt208") if mode == "nt" else ("tn64" if N <= 64 else "tn256"))
    return dict(name="f32_%s_%dx%dx%d%s_ldc%d" % (mode, M, N, K, "_T" if tr else "", ldc), mode=mode, M=M, N=N, K=K, out="f32",
                out_cols=N, ldc=ldc, lda=lda, ldb=ldb, bias=False, act=0, slope=0.2, aux=0, dot=False, sse=False, pad_one=False,
                transpose=tr, tile=tile, split=split, group="f32_" + mode, seed=200 + i)


F32_CASES = [_f32_case(i, *c) for i, c in enumerate(F32)]


def _kind(c):
    """the plan kind plan_gemm picks: 128x64 when the covered columns fit 64, else 128x208 (NT) / 128x256 (TN)"""
    if c["mode"] == "nt":
        return KINDS["nt64"] if max(c["out_cols"], c["N"]) <= 64 else KINDS["nt208"]
    return KINDS["tn64"] if c["N"] <= 64 else KINDS["tn256"]


# ------------------------------------------------------------------ operands, launch, reference
def _nan(rows, cols):
    return torch.full((rows, cols), float("nan"), device="cuda", dtype=torch.bfloat16)


def _tensors(c):
    """seeded operands with bf16 NaN in every element outside the logical extents, prefilled outputs"""
    g = torch.Generator(device="cuda").manual_seed(c["seed"])
    M, N, K = c["M"], c["N"], c["K"]
    T = {}
    if c["mode"] == "nt":
        T["A"], T["B"] = _nan(M + 5, c["lda"]), _nan(N + 5, c["ldb"])
        T["A"][:M, :K] = torch.randn(M, K, device="cuda", generator=g).to(torch.bfloat16)
        T["B"][:N, :K] = (torch.randn(N, K, device="cuda", generator=g) / math.sqrt(K)).to(torch.bfloat16)
    else:
        T["A"], T["B"] = _nan(K + 5, c["lda"]), _nan(K + 5, c["ldb"])
        T["A"][:K, :M] = torch.randn(K, M, device="cuda", generator=g).to(torch.bfloat16)
        T["B"][:K, :N] = (torch.randn(K, N, device="cuda", generator=g) / math.sqrt(K)).to(torch.bfloat16)
    T["bias"] = 0.5 * torch.randn(N, device="cuda", generator=g) if c["bias"] else None
    oc = c["out_cols"]
    if c["aux"]:
        T["aux"] = _nan(M + 5, oc + 8)
        if c["aux"] == 2:       # post-ReLU activations: about half of them exact zeros
            T["aux"][:M, :N] = torch.relu(torch.randn(M, N, device="cuda", generator=g)).to(torch.bfloat16)
        else:                   # sigmoid outputs (aux 1) or targets x in [0, 1] (aux 3)
            T["aux"][:M, :N] = torch.rand(M, N, device="cuda", generator=g).to(torch.bfloat16)
    T["dot_w"] = torch.randn(N, device="cuda", generator=g) if c["dot"] else None
    if c["out"] == "bf16":
        T["out"] = torch.full((M + 3, c["ldc"]), PAT16, device="cuda", dtype=torch.int16).view(torch.bfloat16)
        if c["dot"] or c["sse"]:
            bn = 64 if max(oc, N) <= 64 else 208
            T["slots"] = torch.full((2 * -(-oc // bn), M + 5), PAT32, device="cuda", dtype=torch.int32).view(torch.float32)
    else:
        rows = N if c["transpose"] else M
        T["out"] = torch.full((rows + 2, c["ldc"]), PAT32, device="cuda", dtype=torch.int32).view(torch.float32)
    return T


def _launch(c, T):
    import gm_b200
    kw = dict(M=c["M"], N=c["N"], K=c["K"], transpose=c["transpose"])
    if c["out"] == "bf16":
        kw.update(out_cols=c["out_cols"], pad_one=c["pad_one"], bias=T["bias"], act=c["act"], act_slope=c["slope"],
                  aux=T.get("aux"), aux_mode=c["aux"], dot_w=T["dot_w"], dot_out=T.get("slots"))
    gm_b200.gemm_bf16(T["A"], T["B"], T["out"], c["mode"], **kw)


def _run(c):
    T = _tensors(c)
    _launch(c, T)
    torch.cuda.synchronize()
    return T


def _run_counted(c):
    """-> (tensors, launches per plan kind, library launches): the GEMM under prof_enable(1)"""
    import gm_b200
    T = _tensors(c)
    torch.cuda.synchronize()
    n0 = gm_b200.launch_count()
    gm_b200.prof_enable(1)
    try:
        _launch(c, T)
        counts = [r[3] for r in gm_b200.prof_collect()]
    finally:
        gm_b200.prof_enable(0)
    return T, counts, gm_b200.launch_count() - n0


def _operands64(c, T):
    M, N, K = c["M"], c["N"], c["K"]
    if c["mode"] == "nt":
        return T["A"][:M, :K].double(), T["B"][:N, :K].double()
    return T["A"][:K, :M].double().t(), T["B"][:K, :N].double().t()


def _reference(c, T):
    """float64 A B^T (+ bias) and the accumulation bound e"""
    a, b = _operands64(c, T)
    pre, S = a @ b.t(), a.abs() @ b.abs().t()
    if T["bias"] is not None:
        pre, S = pre + T["bias"].double(), S + T["bias"].double().abs()
    return pre, C_ACC * math.ceil(c["K"] / 16) * 2.0 ** -23 * S


def _ratio(err, tol):
    """worst err / tol; where tol is 0 only an exact match passes"""
    r = torch.where(tol > 0, err / tol.clamp_min(1e-300), torch.where(err > 0, torch.full_like(err, math.inf), torch.zeros_like(err)))
    return float(r.max()) if r.numel() else 0.0


def _activation(c, pre, e):
    """f(pre) of the activation and the error m it may carry from the accumulation"""
    act = c["act"]
    if act == 1:
        return pre.clamp_min(0), e
    if act == 2:
        return torch.sigmoid(pre), 0.25 * e + E_SIG
    if act == 3:
        return torch.where(pre > 0, pre, c["slope"] * pre), max(1.0, abs(c["slope"])) * e
    return pre, e


_WORST = {}


def _record(group, name, ratio):
    if ratio >= _WORST.get(group, (-1.0, ""))[0]:
        _WORST[group] = (ratio, name)
        _REPORT.add(group, {"worst_ratio": ratio, "case": name})


def _check_bf16(c, T):
    """bound on every element and the exact structural checks of one bf16 case -> {group: worst ratio}"""
    M, N, oc = c["M"], c["N"], c["out_cols"]
    out = T["out"]
    pre, e = _reference(c, T)
    fr, m = _activation(c, pre, e)
    act_val, act_m = fr, m
    if c["aux"]:
        a = T["aux"][:M, :N].double()
        if c["aux"] == 1:
            g = a * (1 - a)
            fr, m = fr * g, m * g.abs()
        elif c["aux"] == 2:
            on = (a > 0).double()
            fr, m = fr * on, m * on
        else:   # v = sigmoid output, a = target x: -2 (x - v) v (1 - v), Lipschitz in v on [0, 1]: 0.5 + 2 (|x| + 1)
            fr, m = -2 * (a - fr) * fr * (1 - fr), (0.5 + 2 * (a.abs() + 1)) * m
    m = m + E_OPS * fr.abs()
    got = out[:M, :N].double()
    assert bool(torch.isfinite(out[:M, :oc]).all()), c["name"]
    ratios = {c["group"]: _ratio((got - fr).abs(), U_BF16 * (fr.abs() + m) + m)}
    # padding columns: exact 0, column N exactly 1 under pad_one
    pad = torch.zeros(M, oc - N, device="cuda", dtype=torch.float64)
    if c["pad_one"]:
        pad[:, 0] = 1
    assert torch.equal(out[:M, N:oc].double(), pad), c["name"]
    # rows >= M and columns [out_cols, ldc) keep the prefill bit for bit
    bits = out.view(torch.int16)
    assert bool((bits[M:] == PAT16).all()) and bool((bits[:, oc:] == PAT16).all()), c["name"]
    if c["aux"] == 2:
        assert bool((got[T["aux"][:M, :N] <= 0] == 0).all()), c["name"]
    if c["dot"] or c["sse"]:
        slots = T["slots"]
        assert bool((slots.view(torch.int32)[:, M:] == PAT32).all()), c["name"]
        assert bool(torch.isfinite(slots[:, :M]).all()), c["name"]
        s = slots[:, :M].double().sum(0)
        if c["dot"]:
            w = T["dot_w"].double()
            terms = act_val * w
            ref = terms.sum(1)
            tol = ((act_m + E_OPS * act_val.abs()) * w.abs()).sum(1) + N * 2.0 ** -24 * terms.abs().sum(1)
            ratios["row_dot"] = _ratio((s - ref).abs(), tol)
        else:
            x = T["aux"][:M, :N].double()
            sq = (x - act_val) ** 2
            tol = (2 * (x.abs() + 1) * act_m).sum(1) + (N + 8) * 2.0 ** -24 * sq.sum(1)
            ratios["sse"] = _ratio((s - sq.sum(1)).abs(), tol)
    return ratios


def _check_f32(c, T):
    M, N = c["M"], c["N"]
    pre, e = _reference(c, T)
    out = T["out"]
    rows, cols = (N, M) if c["transpose"] else (M, N)
    got = out[:rows, :cols].double()
    if c["transpose"]:
        got = got.t()
    bits = out.view(torch.int32)
    assert bool((bits[rows:] == PAT32).all()) and bool((bits[:, cols:] == PAT32).all()), c["name"]
    return {c["group"]: _ratio((got - pre).abs(), e)}


def _check(c, T):
    ratios = _check_bf16(c, T) if c["out"] == "bf16" else _check_f32(c, T)
    for grp, r in ratios.items():
        _record(grp, c["name"], r)
    bad = {k: v for k, v in ratios.items() if not v < 1}
    assert not bad, (c["name"], bad)


# ------------------------------------------------------------------ the cases
@pytest.mark.parametrize("c", BF16_CASES, ids=[c["name"] for c in BF16_CASES])
def test_bf16_epilogue_matches_float64(c):
    T, counts, _ = _run_counted(c)
    assert counts == [int(k == KINDS[c["tile"]]) for k in range(4)], (c["name"], counts)
    _check(c, T)


@pytest.mark.parametrize("c", F32_CASES, ids=[c["name"] for c in F32_CASES])
def test_fp32_output_matches_float64(c):
    T, counts, launches = _run_counted(c)
    assert counts == [int(k == KINDS[c["tile"]]) for k in range(4)], (c["name"], counts)
    assert launches == (2 if c["split"] else 1), (c["name"], launches)      # split-K adds the reduction
    _check(c, T)


def _case_from_call(i, A, B, out, mode="nt", N=None, K=None, M=None, act=0, act_slope=0.2, transpose=False, out_cols=None, **rest):
    assert not any(v is not None and v is not False and v != 0 for v in rest.values()), rest   # the conv path: no bias / aux / dot
    if mode == "nt":
        M, N, K = M or A.shape[0], N or B.shape[0], K or A.shape[1]
    else:
        K, M, N = K or A.shape[0], M or A.shape[1], N or B.shape[1]
    f32 = out.dtype == torch.float32
    c = dict(name="dcgan%d_%s_%dx%dx%d" % (i, mode, M, N, K), mode=mode, M=M, N=N, K=K, out="f32" if f32 else "bf16",
             out_cols=N if f32 else (out_cols or N), ldc=out.stride(0), lda=A.stride(0), ldb=B.stride(0), bias=False, act=act,
             slope=act_slope, aux=0, dot=False, sse=False, pad_one=False, transpose=bool(transpose), group="dcgan", seed=300 + i)
    c["tile"] = [k for k, v in KINDS.items() if v == _kind(c)][0]
    return c


def test_dcgan_gemm_calls_match_float64(monkeypatch):
    """every gm_gemm_bf16 call of one d_grad + g_grad of DcganEngine(hidden 64, z 100) at batch 64, replayed with its shapes,
    leading dimensions and epilogue on fresh seeded operands; and conv 1 of D at the benchmark's batch of 1024"""
    import gm_b200
    import gm_b200.dcgan as dcgan
    calls = []
    real = dcgan.gemm_bf16

    def rec(A, B, out, mode="nt", **kw):
        calls.append(_case_from_call(len(calls), A, B, out, mode, **kw))
        return real(A, B, out, mode, **kw)

    monkeypatch.setattr(dcgan, "gemm_bf16", rec)
    eng = gm_b200.DcganEngine(hidden_dim=64, z_dim=100)
    g = torch.Generator().manual_seed(1)
    n = 64
    eng.d_grad(eng.stage_images(torch.rand(n, 3 * 4096, generator=g).cuda()), n, noise=torch.randn(n, 100, generator=g).cuda())
    eng.g_grad(n, noise=torch.randn(n, 100, generator=g).cuda())
    torch.cuda.synchronize()
    monkeypatch.setattr(dcgan, "gemm_bf16", real)
    del eng
    key = lambda c: tuple(v for k, v in sorted(c.items()) if k not in ("name", "seed"))
    uniq = list({key(c): c for c in calls}.values())
    assert len(calls) >= 20 and any(c["act"] == 3 for c in uniq) and any(c["out"] == "f32" for c in uniq), len(calls)
    conv1 = dict(uniq[0], name="dcgan_conv1_bench_batch", mode="nt", M=1 << 20, N=64, K=48, out="bf16", out_cols=64, ldc=64, lda=48,
                 ldb=48, act=3, slope=0.2, transpose=False, tile="nt64", seed=399)
    for c in uniq + [conv1]:
        T, counts, _ = _run_counted(c)
        assert counts == [int(k == KINDS[c["tile"]]) for k in range(4)], (c["name"], counts)
        _check(c, T)
        del T


# ------------------------------------------------------------------ routes that share one mainloop
@pytest.mark.parametrize("tile,N,oc", [("nt208", 400, 416), ("nt64", 64, 64)])
def test_epilogue_routes_agree(tile, N, oc):
    """the universal epilogue (run-time choice, coalesced STG store, register aux loads) against the compile-time
    specialised ones (TMA store, cp.async aux) of the same product: LeakyReLU(0) + bias == ReLU + bias as floats (-0 and
    +0 differ), LeakyReLU(1) == plain bit for bit, aux 1 / aux 2 with a zero bias == without bias as floats"""
    base = dict(name="routes_" + tile, mode="nt", M=1005, N=N, K=784, out="bf16", out_cols=oc, ldc=oc, lda=792, ldb=792, bias=False,
                act=0, slope=0.2, aux=0, dot=False, sse=False, pad_one=False, transpose=False, tile=tile, seed=7)

    def out(**kw):
        c = dict(base, **kw)
        T = _tensors(c)
        if kw.get("zero_bias"):
            T["bias"] = torch.zeros(N, device="cuda")
        _launch(c, T)
        torch.cuda.synchronize()
        return T["out"]

    assert torch.equal(out(bias=True, act=3, slope=0.0).float(), out(bias=True, act=1).float())
    assert torch.equal(out(act=3, slope=1.0).view(torch.int16), out().view(torch.int16))
    for aux in (1, 2):
        assert torch.equal(out(aux=aux, zero_bias=True).float(), out(aux=aux).float()), aux


def test_repeated_calls_give_identical_bits():
    picks = [c for c in BF16_CASES if c["name"] in ("bias_relu_dot_padone_nt208", "bias_sigmoid_aux3_nt64", "lrelu_nt208")]
    picks += [c for c in F32_CASES if c["split"]][:3]
    for c in picks:
        T1, T2 = _run(c), _run(c)
        assert torch.equal(T1["out"].view(torch.int16), T2["out"].view(torch.int16)), c["name"]
        if "slots" in T1:
            assert torch.equal(T1["slots"].view(torch.int32), T2["slots"].view(torch.int32)), c["name"]


def _outputs():
    res = {}
    for c in BF16_CASES + F32_CASES:
        T = _run(c)
        res[c["name"]] = T["out"].view(torch.int16).cpu().numpy()
        if "slots" in T:
            res[c["name"] + "__slots"] = T["slots"].view(torch.int32).cpu().numpy()
    return res


def _dump(path):
    np.savez(path, **_outputs())


@pytest.mark.parametrize("switch", ["GM_NO_TMA_STORE", "GM_NO_PDL"])
def test_outputs_do_not_depend_on_tma_store_or_pdl(switch, tmp_path):
    """every bf16 and fp32 case again in a fresh process with the bulk-tensor store (coalesced stores instead) or the
    programmatic launch serialisation turned off: the same bits"""
    path = str(tmp_path / "out.npz")
    env = dict(os.environ, **{switch: "1"})
    paths = [ROOT, os.path.join(ROOT, "generative-models_b200"), os.path.join(ROOT, "tests")]
    env["PYTHONPATH"] = os.pathsep.join(paths + ([env["PYTHONPATH"]] if env.get("PYTHONPATH") else []))
    code = "import test_gemm_conformance_gpu as T; T._dump(%r)" % path
    r = subprocess.run([sys.executable, "-c", code], env=env, cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    other = np.load(path)
    mine = _outputs()
    assert sorted(other.files) == sorted(mine)
    diff = [k for k in mine if not np.array_equal(mine[k], other[k])]
    assert not diff, diff


def test_dependent_chain_without_host_sync():
    """bf16 -> bf16 -> TN fp32 split-K -> reduction enqueued back to back: each stage against float64 of the stored output
    of the stage before (prefilled with NaN, so a read ahead of its producer shows)"""
    import gm_b200
    M, K, H1, H2 = 4096, 784, 400, 208
    g = torch.Generator(device="cuda").manual_seed(21)
    X = torch.randn(M, K, device="cuda", generator=g).to(torch.bfloat16)
    W1 = (torch.randn(H1, K, device="cuda", generator=g) / math.sqrt(K)).to(torch.bfloat16)
    b1 = 0.5 * torch.randn(H1, device="cuda", generator=g)
    W2 = (torch.randn(H2, H1, device="cuda", generator=g) / math.sqrt(H1)).to(torch.bfloat16)
    h1, h2 = _nan(M, 416), _nan(M, H2)
    gw = torch.full((H1, 256), float("nan"), device="cuda")
    torch.cuda.synchronize()
    n0 = gm_b200.launch_count()
    gm_b200.gemm_bf16(X, W1, h1, "nt", bias=b1, act=1, pad_one=True, out_cols=416)
    gm_b200.gemm_bf16(h1, W2, h2, "nt", K=H1)
    gm_b200.gemm_bf16(h1, h2, gw, "tn", M=H1, N=H2, K=M)
    torch.cuda.synchronize()
    assert gm_b200.launch_count() - n0 == 4                                    # the fp32 product ran split-K
    x64, h164, h264 = X.double(), h1[:, :H1].double(), h2.double()
    worst = 0.0
    pre = x64 @ W1.double().t() + b1.double()
    e = C_ACC * math.ceil(K / 16) * 2.0 ** -23 * (x64.abs() @ W1.double().abs().t() + b1.double().abs())
    fr = pre.clamp_min(0)
    worst = max(worst, _ratio((h164 - fr).abs(), U_BF16 * (fr.abs() + e) + e))
    pre = h164 @ W2.double().t()
    e = C_ACC * math.ceil(H1 / 16) * 2.0 ** -23 * (h164.abs() @ W2.double().abs().t())
    worst = max(worst, _ratio((h264 - pre).abs(), U_BF16 * (pre.abs() + e) + e))
    pre = h164.t() @ h264
    e = C_ACC * math.ceil(M / 16) * 2.0 ** -23 * (h164.abs().t() @ h264.abs())
    worst = max(worst, _ratio((gw[:, :H2].double() - pre).abs(), e))
    _record("chain", "bf16_bf16_tn_splitk", worst)
    assert worst < 1, worst
    assert bool(torch.isnan(gw[:, H2:]).all())                               # the reduction writes the logical columns only


# ------------------------------------------------------------------ descriptors the library refuses
def test_invalid_descriptors_are_refused_before_any_launch():
    import ctypes as C
    from gm_b200 import _lib
    M, N, K = 64, 32, 64
    A = torch.zeros(M, K, device="cuda", dtype=torch.bfloat16)
    B = torch.zeros(N, K, device="cuda", dtype=torch.bfloat16)
    ob = torch.zeros(M + 1, 64, device="cuda", dtype=torch.bfloat16)
    of = torch.zeros(M + 1, 64, device="cuda")
    aux = torch.zeros(M + 1, 64, device="cuda", dtype=torch.bfloat16)
    vec = torch.zeros(68, device="cuda")
    slots = torch.zeros(2, M, device="cuda")

    def desc(**kw):
        d = _lib.GemmDesc()
        d.mode, d.M, d.N, d.K = 0, M, N, K
        d.A, d.lda, d.B, d.ldb = A.data_ptr(), K, B.data_ptr(), K
        d.out_kind, d.Cp, d.ldc, d.out_cols = 0, ob.data_ptr(), 64, N
        d.act_slope = 0.2
        for k, v in kw.items():
            setattr(d, k, v)
        return d

    f32 = dict(out_kind=1, Cp=of.data_ptr())
    bad = {
        "mode 2": desc(mode=2), "mode -1": desc(mode=-1),
        "TN with a bf16 output": desc(mode=1),
        "act 4": desc(act=4), "act -1": desc(act=-1),
        "aux_mode 4 (AUX_L1)": desc(aux=aux.data_ptr(), ld_aux=64, aux_mode=4), "aux_mode 5": desc(aux=aux.data_ptr(), ld_aux=64, aux_mode=5),
        "aux_mode without aux": desc(aux_mode=1), "aux without aux_mode": desc(aux=aux.data_ptr(), ld_aux=64),
        "out_kind 2": desc(out_kind=2),
        "fp32 with bias": desc(bias=vec.data_ptr(), **f32), "fp32 with act": desc(act=1, **f32),
        "fp32 with pad_one": desc(pad_one=1, **f32), "fp32 with out_cols": desc(out_cols=48, **f32),
        "fp32 with aux": desc(aux=aux.data_ptr(), ld_aux=64, aux_mode=1, **f32),
        "fp32 with dot": desc(dot_w=vec.data_ptr(), dot_out=slots.data_ptr(), dot_ld=M, **f32),
        "fp32 ldc below N": desc(ldc=N - 1, **f32), "fp32 transposed ldc below M": desc(transpose=1, ldc=M - 1, **f32),
        "bf16 transpose": desc(transpose=1),
        "bf16 ldc % 8": desc(ldc=36), "bf16 ldc below out_cols": desc(ldc=40, out_cols=48),
        "bf16 out_cols % 8": desc(out_cols=36), "ld_aux % 8": desc(aux=aux.data_ptr(), ld_aux=60, aux_mode=2),
        "ld_aux below out_cols": desc(aux=aux.data_ptr(), ld_aux=24, aux_mode=2),
        "C misaligned": desc(Cp=ob.data_ptr() + 2), "fp32 C misaligned": desc(Cp=of.data_ptr() + 4, ldc=60, **{"out_kind": 1}),
        "aux misaligned": desc(aux=aux.data_ptr() + 2, ld_aux=64, aux_mode=2),
        "bias misaligned": desc(bias=vec.data_ptr() + 4), "dot_w misaligned": desc(dot_w=vec.data_ptr() + 4, dot_out=slots.data_ptr(), dot_ld=M),
        "dot_w without dot_out": desc(dot_w=vec.data_ptr()), "dot_ld below M": desc(dot_w=vec.data_ptr(), dot_out=slots.data_ptr(), dot_ld=M - 1),
    }
    h = _lib.ctx()
    L = _lib.lib()
    torch.cuda.synchronize()
    n0 = L.gm_launch_count(h, 0)
    for what, d in bad.items():
        rc = L.gm_gemm_bf16(h, C.byref(d), _lib._stream())
        assert rc != 0 and L.gm_last_error(h).decode(), what
        with pytest.raises(_lib.GmError):
            _lib.check(h, rc)
    assert L.gm_launch_count(h, 0) == n0
    # the valid neighbours of those descriptors still run
    for d in (desc(), desc(**f32), desc(out_kind=1, Cp=of.data_ptr(), out_cols=0), desc(act=3, bias=vec.data_ptr()),
              desc(dot_w=vec.data_ptr(), dot_out=slots.data_ptr(), dot_ld=M)):
        _lib.check(h, L.gm_gemm_bf16(h, C.byref(d), _lib._stream()))
    torch.cuda.synchronize()
    assert L.gm_launch_count(h, 0) == n0 + 5
