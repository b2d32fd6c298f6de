"""Sliding-window wgmma attention (the WIN kernels) against the fp32 reference with the window mask, alone and combined
with document masking; bit-identity when the window covers the sequence; block skipping shown with NaN rows; the
refused window; and a ``debug-mistral`` training step against an fp32 model."""
import math
import os
import subprocess
import sys
from pathlib import Path

import pytest
import torch

from distributed_training_guide_b200 import _ext, ops
from distributed_training_guide_b200.ops import reference as ref
from test_gpu_attention import FWD_TILE_TOL, GRAD_TILE_TOL, LSE_TOL, _assert_tiles, _grad_slices
from test_gpu_attention_docmask import _doc_start
from test_gpu_step_reference import LOSS_FACTOR, LOSS_SLACK, _capture_buckets, _check_grads, _engine_grads, _fp32_matmuls

pytestmark = pytest.mark.gpu
DEV = "cuda"
ROOT = Path(__file__).resolve().parents[1]
SC = 1.0 / math.sqrt(128)


def _ref(qkv, do, nh, nkv, scale, window, ds=None):
    """fp32 output, natural-log lse and d(qkv) of attention with a sliding window (and document masking)."""
    qf = qkv.detach().float().requires_grad_(True)
    q, k, v = qf[:, :, :nh], qf[:, :, nh:nh + nkv], qf[:, :, nh + nkv:]
    o = ref.attention(q, k, v, scale=scale, doc_start=ds, window=window)
    o.backward(do.float())
    with torch.no_grad():
        kr = k.permute(0, 2, 1, 3).repeat_interleave(nh // nkv, 1)
        S = qkv.shape[1]
        lse = torch.empty(qkv.shape[0], nh, S, device=DEV)
        mask = ref.document_mask(ds, S, window, device=DEV)
        for r0 in range(0, S, 512):
            s = (q[:, r0:r0 + 512].permute(0, 2, 1, 3) @ kr.transpose(-1, -2)) * scale
            lse[:, :, r0:r0 + 512] = torch.logsumexp(s.masked_fill(~mask[:, None, r0:r0 + 512], float("-inf")), -1)
    return o.detach(), lse, qf.grad


def _check(qkv, do, nh, nkv, window, ds=None):
    C = _ext.load(True)
    want_o, want_lse, want_g = _ref(qkv, do, nh, nkv, SC, window, ds)
    for version in (1, 2):
        o, lse = C.attn_fwd(qkv, nh, nkv, SC, version, doc_start=ds, window=window)
        _assert_tiles(f"W {window} forward v{version}", o, want_o, FWD_TILE_TOL)
        err = (lse - want_lse).abs().max().item()
        assert err < LSE_TOL, f"W {window} forward v{version}: lse max err {err:.4g}"
        if window == 1 and ds is None:   # a query that sees only itself returns its own v
            assert torch.equal(o, qkv[:, :, nh + nkv:].repeat_interleave(nh // nkv, 2))
    for mode in (1, 2):
        g = C.attn_bwd(do, qkv, o, lse, nh, nkv, SC, None, mode, doc_start=ds, window=window)
        for name, sl in _grad_slices(nh, nkv):
            if window == 1 and name != "dv":
                # P = 1 and dP = delta exactly, so dQ and dK are 0 up to the rounding of two fp32 dot products of
                # the same terms
                assert g[:, :, sl].float().abs().max().item() < 1e-3, f"W 1 mode {mode} {name}"
            else:
                _assert_tiles(f"W {window} mode {mode} {name}", g[:, :, sl], want_g[:, :, sl], GRAD_TILE_TOL)


@pytest.mark.parametrize("nh,nkv", [(2, 2), (4, 1)])
@pytest.mark.parametrize("S", [128, 384, 1024, 4096])
@pytest.mark.parametrize("w", [1, 64, 127, 128, 129, 192, 1000, "S-1", "S", "2S"])
def test_window_forward_and_backward_against_reference(w, S, nh, nkv):
    window = {"S-1": S - 1, "S": S, "2S": 2 * S}.get(w, w)
    torch.manual_seed(0)
    qkv = torch.randn(2, S, nh + 2 * nkv, 128, device=DEV, dtype=torch.bfloat16)
    do = torch.randn(2, S, nh, 128, device=DEV, dtype=torch.bfloat16)
    _check(qkv, do, nh, nkv, window)


@pytest.mark.parametrize("S,nh,nkv,window", [(1024, 4, 1, 192), (1024, 2, 2, 129), (4096, 8, 2, 1000),
                                             (4096, 4, 1, 128)])
def test_window_with_document_masking(S, nh, nkv, window):
    """Documents both shorter and longer than the window, a different layout per row."""
    torch.manual_seed(1)
    rows = [[0, 50, 51, 600, 700, 1000, 3000], [0, 1, 63, 64, 129, 900, 2500, 2600]]
    ds = torch.stack([_doc_start(S, [c for c in r if c < S]) for r in rows]).to(DEV)
    qkv = torch.randn(2, S, nh + 2 * nkv, 128, device=DEV, dtype=torch.bfloat16)
    do = torch.randn(2, S, nh, 128, device=DEV, dtype=torch.bfloat16)
    _check(qkv, do, nh, nkv, window, ds)


@pytest.mark.parametrize("docs", [False, True])
def test_window_covering_the_sequence_is_bit_identical(docs):
    C = _ext.load(True)
    torch.manual_seed(2)
    S, nh, nkv = 1024, 4, 2
    qkv = torch.randn(2, S, nh + 2 * nkv, 128, device=DEV, dtype=torch.bfloat16)
    do = torch.randn(2, S, nh, 128, device=DEV, dtype=torch.bfloat16)
    ds = torch.stack([_doc_start(S, [0, 100, 700])] * 2).to(DEV) if docs else None
    for version in (1, 2):
        o0, l0 = C.attn_fwd(qkv, nh, nkv, SC, version, doc_start=ds)
        for window in (S, S + 1, 2 * S, 2 ** 31 - 1):
            o1, l1 = C.attn_fwd(qkv, nh, nkv, SC, version, doc_start=ds, window=window)
            assert torch.equal(o0, o1) and torch.equal(l0, l1), (version, window)
        for mode in (1, 2):
            g0 = C.attn_bwd(do, qkv, o0, l0, nh, nkv, SC, None, mode, doc_start=ds)
            g1 = C.attn_bwd(do, qkv, o0, l0, nh, nkv, SC, None, mode, doc_start=ds, window=S)
            assert torch.equal(g0, g1), (version, mode)


@pytest.mark.parametrize("window", [128, 192, 1000])
def test_queries_beyond_the_window_skip_a_nan_key(window):
    """One key row of K and V is NaN.  A loaded-but-masked V block would turn 0 * NaN into NaN, so queries more than
    W + 255 tokens after it stay finite in O and dQ only if the kernels skip its blocks; the causal kernels make them
    NaN."""
    C = _ext.load(True)
    torch.manual_seed(3)
    S, nh, nkv, kn = 2048, 4, 2, 300
    qkv = torch.randn(1, S, nh + 2 * nkv, 128, device=DEV, dtype=torch.bfloat16)
    qkv[:, kn, nh:] = float("nan")
    do = torch.randn(1, S, nh, 128, device=DEV, dtype=torch.bfloat16)
    far = kn + window + 256
    for version in (1, 2):
        o, lse = C.attn_fwd(qkv, nh, nkv, SC, version, window=window)
        assert torch.isfinite(o[:, far:]).all() and torch.isfinite(lse[:, :, far:]).all(), version
        assert torch.isnan(o[:, kn:kn + window]).all(), version     # the rows that do see the key
        # tiles before the key's block never load it (the earlier rows of its own tile do: the diagonal block)
        assert torch.isfinite(o[:, :kn // 128 * 128]).all(), version
        oc, _ = C.attn_fwd(qkv, nh, nkv, SC, version)
        assert torch.isnan(oc[:, far:]).all(), version
        for mode in (1, 2):
            g = C.attn_bwd(do, qkv, o, lse, nh, nkv, SC, None, mode, window=window)
            assert torch.isfinite(g[:, far:, :nh]).all(), (version, mode)


@pytest.mark.parametrize("window", [128, 192, 1000])
def test_keys_before_the_window_skip_a_nan_query(window):
    """One query row of Q and dO is NaN.  Keys more than W + 255 tokens before it get finite dK / dV only if the
    dK / dV pass stops before that query's block; the causal kernels make them NaN."""
    C = _ext.load(True)
    torch.manual_seed(4)
    S, nh, nkv, qn = 2048, 4, 2, 1800
    qkv = torch.randn(1, S, nh + 2 * nkv, 128, device=DEV, dtype=torch.bfloat16)
    do = torch.randn(1, S, nh, 128, device=DEV, dtype=torch.bfloat16)
    qkv[:, qn, :nh] = float("nan")
    do[:, qn] = float("nan")
    near = qn - window - 255
    for version in (1, 2):
        o, lse = C.attn_fwd(qkv, nh, nkv, SC, version, window=window)
        oc, lc = C.attn_fwd(qkv, nh, nkv, SC, version)
        for mode in (1, 2):
            g = C.attn_bwd(do, qkv, o, lse, nh, nkv, SC, None, mode, window=window)
            assert torch.isfinite(g[:, :near, nh:]).all(), (version, mode)
            assert torch.isnan(g[:, qn - window + 1:qn + 1, nh:]).all(), (version, mode)   # keys the query sees
            gc = C.attn_bwd(do, qkv, oc, lc, nh, nkv, SC, None, mode)
            assert torch.isnan(gc[:, :near, nh:]).all(), (version, mode)


def _refused(call, match):
    torch.cuda.synchronize()
    n0 = _ext.launch_count()
    with pytest.raises(RuntimeError, match=match):
        call()
    assert _ext.launch_count() == n0, "a refused call launched a kernel"


def test_binding_refuses_window_below_one():
    C = _ext.load(True)
    S, nh, nkv = 256, 2, 1
    qkv = torch.randn(1, S, nh + 2 * nkv, 128, device=DEV, dtype=torch.bfloat16)
    do = torch.randn(1, S, nh, 128, device=DEV, dtype=torch.bfloat16)
    o, lse = C.attn_fwd(qkv, nh, nkv, SC)
    for bad in (0, -1, -(2 ** 40)):
        _refused(lambda: C.attn_fwd(qkv, nh, nkv, SC, 1, window=bad), "window")
        _refused(lambda: C.attn_fwd(qkv, nh, nkv, SC, 2, window=bad), "window")
        _refused(lambda: C.attn_bwd(do, qkv, o, lse, nh, nkv, SC, None, 1, window=bad), "window")
        _refused(lambda: C.attn_bwd(do, qkv, o, lse, nh, nkv, SC, None, 2, window=bad), "window")


def test_attention_qkv_window_through_autograd_and_sdpa_fallback():
    """``ops.attention_qkv(window=...)`` on the kernels (S % 128 == 0) and on the SDPA fallback (S 200)."""
    torch.manual_seed(5)
    nh, nkv = 4, 2
    for S, window in ((512, 192), (200, 50)):
        qkv = torch.randn(1, S, nh + 2 * nkv, 128, device=DEV, dtype=torch.bfloat16, requires_grad=True)
        do = torch.randn(1, S, nh, 128, device=DEV, dtype=torch.bfloat16)
        o = ops.attention_qkv(qkv * 1.0, nh, nkv, window=window)
        o.backward(do)
        want_o, _, want_g = _ref(qkv, do, nh, nkv, SC, window)
        assert (o.float() - want_o).abs().max().item() < 2e-2, S
        assert (qkv.grad.float() - want_g).abs().max().item() < 5e-2, S


# ------------------------------------------------------------------------------------------------------------------
# a debug-mistral training step against an fp32 model
# ------------------------------------------------------------------------------------------------------------------
def _plain_grads(config, weights, batch, dtype, monkeypatch):
    from distributed_training_guide_b200.models.llama import build_llama

    model = build_llama(config, dtype=dtype, device="cuda", init=False)
    with torch.no_grad():
        for n, p in model.named_parameters():
            p.copy_(weights[n])
    with monkeypatch.context() as mp, _fp32_matmuls():
        if dtype == torch.bfloat16:
            mp.setattr(_ext, "_forced", {"all"})
        out = model(**{k: v.cuda() for k, v in batch.items()})
        out.loss.backward()
    return out.loss.item(), {n: p.grad.float() for n, p in model.named_parameters()}


def test_mistral_step_matches_fp32_reference(monkeypatch):
    from distributed_training_guide_b200.engine import TrainEngine

    B, S = 2, 512   # beyond debug-mistral's window of 192
    eng = TrainEngine.create("debug-mistral", parallelism="single", batch_size=B, seq_length=S, lr=5e-3,
                             device="cuda")
    try:
        assert eng.config.sliding_window == 192
        weights = {n: p.detach().clone() for n, p in eng.model.named_parameters()}
        ids = torch.randint(0, eng.config.vocab_size, (B, S), generator=torch.Generator().manual_seed(7))
        batch = {"input_ids": ids, "labels": ids.clone()}
        rec = _capture_buckets(eng)
        loss = float(eng.step(batch))
        grads = _engine_grads(eng, rec)
    finally:
        eng.close()
    l32, g32 = _plain_grads(eng.config, weights, batch, torch.float32, monkeypatch)
    l16, g16 = _plain_grads(eng.config, weights, batch, torch.bfloat16, monkeypatch)
    assert abs(loss - l32) <= LOSS_FACTOR * abs(l16 - l32) + LOSS_SLACK, (loss, l32, l16)
    _check_grads("mistral", grads, g32, g16, [])


def test_chapter_01_trains_debug_mistral(tmp_path):
    cmd = [sys.executable, str(ROOT / "01-single-gpu" / "train_llm.py"), "-d", "synthetic", "-m", "debug-mistral",
           "-s", "512", "-b", "2", "--max-steps", "4", "--log-freq", "2", "--num-workers", "0",
           "--save-dir", str(tmp_path)]
    r = subprocess.run(cmd, capture_output=True, text=True, cwd=str(ROOT / "01-single-gpu"), timeout=600,
                       env={**os.environ, "PYTHONPATH": str(ROOT)})
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    losses = [float(line.split("'running_loss': ")[1].split(",")[0]) for line in (r.stdout + r.stderr).splitlines()
              if "'running_loss': " in line]
    assert losses and all(math.isfinite(x) for x in losses), losses
