"""Document-masked wgmma attention (the DOC kernels) against the fp32 reference with the mask, bit-identity where
the arithmetic is the same as the plain kernels', block skipping, and a packed-document training step against an
fp32 model."""
import math
import os
import subprocess
import sys
from pathlib import Path

import pytest
import torch

from distributed_training_guide_b200 import _ext, ops
from distributed_training_guide_b200.ops import reference as ref
from distributed_training_guide_b200.utils.data import positions_from_starts
from test_gpu_attention import FWD_TILE_TOL, GRAD_TILE_TOL, LSE_TOL, _assert_tiles, _grad_slices
from test_gpu_step_reference import LOSS_FACTOR, LOSS_SLACK, _capture_buckets, _check_grads, _engine_grads, _fp32_matmuls

pytestmark = pytest.mark.gpu
DEV = "cuda"
ROOT = Path(__file__).resolve().parents[1]


def _doc_start(S, cuts):
    """int32 [S] document starts for documents beginning at ``cuts`` (0 is always a start)."""
    starts = torch.zeros(S, dtype=torch.bool)
    starts[list(cuts)] = True
    return ops.document_starts(positions_from_starts(starts)[None])[0]


def _layouts(B, S, layout):
    if layout == "one":
        rows = [[0]] * B
    elif layout == "aligned":
        rows = [[c for c in (0, 128, 384, 1024, 2048) if c < S]] * B
    elif layout == "midtile":
        rows = [[c for c in (0, 1, 63, 64, 127, 129, 1000) if c < S]] * B
    elif layout == "each-token":
        rows = [list(range(S))] * B
    elif layout == "per-row":   # B = 2 with different layouts per row
        rows = [[c for c in (0, 1, 63, 64, 127, 129, 1000) if c < S], [c for c in (0, 200, 201, 3000) if c < S]]
        rows = (rows * B)[:B]
    else:
        raise ValueError(layout)
    return torch.stack([_doc_start(S, r) for r in rows]).to(DEV)


def _ref(qkv, do, nh, nkv, scale, ds):
    """fp32 output, natural-log lse and d(qkv) of document-masked attention."""
    qf = qkv.detach().float().requires_grad_(True)
    q, k, v = qf[:, :, :nh], qf[:, :, nh:nh + nkv], qf[:, :, nh + nkv:]
    o = ref.attention(q, k, v, scale=scale, doc_start=ds)
    o.backward(do.float())
    with torch.no_grad():
        kr = k.permute(0, 2, 1, 3).repeat_interleave(nh // nkv, 1)
        lse = torch.empty(qkv.shape[0], nh, qkv.shape[1], device=DEV)
        S = qkv.shape[1]
        for r0 in range(0, S, 512):
            s = (q[:, r0:r0 + 512].permute(0, 2, 1, 3) @ kr.transpose(-1, -2)) * scale
            m = ref.document_mask(ds, S)[:, r0:r0 + 512]
            lse[:, :, r0:r0 + 512] = torch.logsumexp(s.masked_fill(~m[:, None], float("-inf")), -1)
    return o.detach(), lse, qf.grad


CASES = [  # (B, S, nh, nkv, layout)
    (1, 128, 2, 1, "midtile"), (1, 384, 4, 2, "aligned"), (1, 384, 4, 4, "midtile"), (2, 384, 4, 2, "per-row"),
    (1, 128, 2, 2, "each-token"), (1, 384, 2, 1, "each-token"), (2, 1024, 8, 2, "per-row"),
    (1, 4096, 32, 8, "midtile"), (1, 4096, 32, 32, "aligned"), (2, 4096, 32, 8, "per-row"),
]


@pytest.mark.parametrize("B,S,nh,nkv,layout", CASES)
def test_docmask_forward_and_backward_against_reference(B, S, nh, nkv, layout):
    torch.manual_seed(0)
    C = _ext.load(True)
    sc = 1.0 / math.sqrt(128)
    qkv = torch.randn(B, S, nh + 2 * nkv, 128, device=DEV, dtype=torch.bfloat16)
    do = torch.randn(B, S, nh, 128, device=DEV, dtype=torch.bfloat16)
    ds = _layouts(B, S, layout)
    want_o, want_lse, want_g = _ref(qkv, do, nh, nkv, sc, ds)
    for version in (1, 2):
        o, lse = C.attn_fwd(qkv, nh, nkv, sc, version, doc_start=ds)
        _assert_tiles(f"forward v{version}", o, want_o, FWD_TILE_TOL)
        err = (lse - want_lse).abs().max().item()
        assert err < LSE_TOL, f"forward v{version}: lse max err {err:.4g}"
        if layout == "each-token":   # a query that sees only itself returns its own v
            assert torch.equal(o, qkv[:, :, nh + nkv:].repeat_interleave(nh // nkv, 2))
    for mode in (1, 2):
        g = C.attn_bwd(do, qkv, o, lse, nh, nkv, sc, None, mode, doc_start=ds)
        for name, sl in _grad_slices(nh, nkv):
            if layout == "each-token" and name != "dv":
                # P = 1 and dP = delta exactly, so dQ and dK are 0 up to the rounding of two fp32 dot products of the
                # same terms; a relative error against the reference's own rounding noise means nothing
                assert g[:, :, sl].float().abs().max().item() < 1e-3, f"mode {mode} {name}"
            else:
                _assert_tiles(f"mode {mode} {name}", g[:, :, sl], want_g[:, :, sl], GRAD_TILE_TOL)


@pytest.mark.parametrize("S,nh,nkv", [(384, 4, 2), (4096, 32, 8)])
def test_one_document_is_bit_identical_to_plain_kernels(S, nh, nkv):
    torch.manual_seed(1)
    C = _ext.load(True)
    sc = 1.0 / math.sqrt(128)
    qkv = torch.randn(2, S, nh + 2 * nkv, 128, device=DEV, dtype=torch.bfloat16)
    do = torch.randn(2, S, nh, 128, device=DEV, dtype=torch.bfloat16)
    ds = _layouts(2, S, "one")
    for version in (1, 2):
        o0, l0 = C.attn_fwd(qkv, nh, nkv, sc, version)
        o1, l1 = C.attn_fwd(qkv, nh, nkv, sc, version, doc_start=ds)
        assert torch.equal(o0, o1) and torch.equal(l0, l1), version
        for mode in (1, 2):
            g0 = C.attn_bwd(do, qkv, o0, l0, nh, nkv, sc, None, mode)
            g1 = C.attn_bwd(do, qkv, o0, l0, nh, nkv, sc, None, mode, doc_start=ds)
            assert torch.equal(g0, g1), (version, mode)


@pytest.mark.parametrize("nh,nkv", [(4, 2), (8, 8)])
def test_aligned_documents_equal_documents_alone_and_skip_other_blocks(nh, nkv):
    """128-aligned documents: each document's O / lse / dQKV slice equals the plain kernels on that document alone,
    bit for bit, with NaN in every other document's q, k, v and dO.  A masked-but-loaded block would turn 0 * NaN into
    NaN, so this shows the blocks are skipped."""
    torch.manual_seed(2)
    C = _ext.load(True)
    sc = 1.0 / math.sqrt(128)
    S, bounds = 1024, [0, 128, 384, 512, 1024]
    qkv = torch.randn(1, S, nh + 2 * nkv, 128, device=DEV, dtype=torch.bfloat16)
    do = torch.randn(1, S, nh, 128, device=DEV, dtype=torch.bfloat16)
    ds = _doc_start(S, bounds[:-1])[None].to(DEV)
    for a, b in zip(bounds[:-1], bounds[1:]):
        x, dx = torch.full_like(qkv, float("nan")), torch.full_like(do, float("nan"))
        x[:, a:b], dx[:, a:b] = qkv[:, a:b], do[:, a:b]
        alone_x, alone_do = qkv[:, a:b].contiguous(), do[:, a:b].contiguous()
        for version in (1, 2):
            o, lse = C.attn_fwd(x, nh, nkv, sc, version, doc_start=ds)
            oa, la = C.attn_fwd(alone_x, nh, nkv, sc, version)
            assert torch.equal(o[:, a:b], oa) and torch.equal(lse[:, :, a:b], la), (a, version)
            for mode in (1, 2):
                g = C.attn_bwd(dx, x, o, lse, nh, nkv, sc, None, mode, doc_start=ds)
                ga = C.attn_bwd(alone_do, alone_x, oa, la, nh, nkv, sc, None, mode)
                assert torch.equal(g[:, a:b], ga), (a, version, mode)


def test_binding_refuses_bad_doc_start():
    C = _ext.load(True)
    qkv = torch.randn(1, 256, 4, 128, device=DEV, dtype=torch.bfloat16)
    good = torch.zeros(1, 256, dtype=torch.int32, device=DEV)
    for bad, msg in [(good.long(), "int32"), (good[:, :128], r"\[B, S\]"), (good.cpu(), "device"),
                     (torch.zeros(1, 512, dtype=torch.int32, device=DEV)[:, ::2], "contiguous")]:
        with pytest.raises(RuntimeError, match=msg):
            C.attn_fwd(qkv, 2, 1, 0.1, doc_start=bad)


def test_out_of_range_doc_start_stays_in_bounds():
    """Starts that no position ids can produce (negative, beyond the token, beyond S) only change values: the block
    indices are clamped, so every read and write stays inside the tensors and the outputs keep their shapes."""
    C = _ext.load(True)
    S, nh, nkv = 512, 2, 1
    qkv = torch.randn(1, S, nh + 2 * nkv, 128, device=DEV, dtype=torch.bfloat16)
    do = torch.randn(1, S, nh, 128, device=DEV, dtype=torch.bfloat16)
    for fill in (-1000, 10 ** 6):
        ds = torch.full((1, S), fill, dtype=torch.int32, device=DEV)
        o, lse = C.attn_fwd(qkv, nh, nkv, 0.1, doc_start=ds)
        g = C.attn_bwd(do, qkv, o, lse, nh, nkv, 0.1, doc_start=ds)
        torch.cuda.synchronize()
        assert o.shape == (1, S, nh, 128) and g.shape == qkv.shape


def test_attention_qkv_sdpa_fallback_honours_doc_start():
    """S % 128 != 0 takes the SDPA path with an explicit mask."""
    torch.manual_seed(4)
    nh, nkv, S = 4, 2, 200
    qkv = torch.randn(1, S, nh + 2 * nkv, 128, device=DEV, dtype=torch.bfloat16)
    ds = _doc_start(S, [0, 50, 51, 120])[None].to(DEV)
    o = ops.attention_qkv(qkv, nh, nkv, doc_start=ds)
    want = ref.attention(qkv[:, :, :nh].float(), qkv[:, :, nh:nh + nkv].float(), qkv[:, :, nh + nkv:].float(),
                         doc_start=ds)
    assert (o.float() - want).abs().max().item() < 2e-2


# ------------------------------------------------------------------------------------------------------------------
# a packed-document training step against an fp32 model with the same mask
# ------------------------------------------------------------------------------------------------------------------
def _plain_grads(config, weights, batch, dtype, monkeypatch):
    from distributed_training_guide_b200.models.llama import build_llama

    model = build_llama(config, dtype=dtype, device="cuda", init=False)
    model.document_masking = True
    with torch.no_grad():
        for n, p in model.named_parameters():
            p.copy_(weights[n])
    with monkeypatch.context() as mp, _fp32_matmuls():
        if dtype == torch.bfloat16:
            mp.setattr(_ext, "_forced", {"all"})
        out = model(**{k: v.cuda() for k, v in batch.items()})
        out.loss.backward()
    return out.loss.item(), {n: p.grad.float() for n, p in model.named_parameters()}


def test_packed_step_matches_fp32_reference(monkeypatch):
    from distributed_training_guide_b200.engine import TrainEngine

    B, S = 2, 512
    eng = TrainEngine.create("debug-llama-gqa", parallelism="single", batch_size=B, seq_length=S, lr=5e-3,
                             device="cuda", document_masking=True)
    try:
        weights = {n: p.detach().clone() for n, p in eng.model.named_parameters()}
        g = torch.Generator().manual_seed(7)
        ids = torch.randint(0, eng.config.vocab_size, (B, S), generator=g)
        starts = torch.zeros(B, S, dtype=torch.bool)
        starts[0, [0, 1, 100, 128, 129, 300]] = True
        starts[1, [0, 256, 257, 511]] = True
        batch = {"input_ids": ids, "labels": ids.clone(), "position_ids": positions_from_starts(starts)}
        rec = _capture_buckets(eng)
        loss = float(eng.step(batch))
        grads = _engine_grads(eng, rec)
    finally:
        eng.close()
    l32, g32 = _plain_grads(eng.config, weights, batch, torch.float32, monkeypatch)
    l16, g16 = _plain_grads(eng.config, weights, batch, torch.bfloat16, monkeypatch)
    assert abs(loss - l32) <= LOSS_FACTOR * abs(l16 - l32) + LOSS_SLACK, (loss, l32, l16)
    report = []
    _check_grads("docmask", grads, g32, g16, report)


def test_chapter_01_trains_with_document_masking(tmp_path):
    cmd = [sys.executable, str(ROOT / "01-single-gpu" / "train_llm.py"), "-d", "synthetic", "-m", "debug-llama-gqa",
           "--document-masking", "-s", "512", "-b", "2", "--max-steps", "4", "--log-freq", "2", "--num-workers", "0",
           "--save-dir", str(tmp_path)]
    r = subprocess.run(cmd, capture_output=True, text=True, cwd=str(ROOT / "01-single-gpu"), timeout=600,
                       env={**os.environ, "PYTHONPATH": str(ROOT)})
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    losses = [float(line.split("'running_loss': ")[1].split(",")[0]) for line in (r.stdout + r.stderr).splitlines()
              if "'running_loss': " in line]
    assert losses and all(math.isfinite(x) for x in losses), losses
