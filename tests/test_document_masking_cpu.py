"""Document masking (``--document-masking``) on the CPU: the ``document_starts`` convention, the masked reference
attention, a packed Llama row against its documents run alone, ``position_ids`` from every data source, the CLI and
the engines that refuse the flag, and DDP / FSDP over gloo against a single process."""
import json

import numpy as np
import pytest
import torch

from dist_utils import run_distributed
from distributed_training_guide_b200 import ops
from distributed_training_guide_b200.ops import reference as ref
from distributed_training_guide_b200.utils import data as data_utils


def _starts_from_lengths(lengths):
    pos = torch.cat([torch.arange(n) for n in lengths])
    return pos, ops.document_starts(pos[None])[0]


# ---------------------------------------------------------------------------------------------------------------
# the convention
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("pos,expect", [
    ([0, 1, 2, 3, 4], [0, 0, 0, 0, 0]),                       # one document
    ([0, 0, 0, 0], [0, 1, 2, 3]),                             # length-1 documents
    ([0, 1, 2, 3, 0], [0, 0, 0, 0, 4]),                       # a boundary at the last token
    ([0, 1, 0, 1, 2, 0, 0, 1, 0, 1], [0, 0, 2, 2, 2, 5, 6, 6, 8, 8]),   # many boundaries
    ([7, 8, 9, 0, 1], [0, 0, 0, 3, 3]),                       # a row that starts mid-document
])
def test_document_starts_on_hand_made_rows(pos, expect):
    got = ops.document_starts(torch.tensor([pos]))
    assert got.dtype == torch.int32 and got.is_contiguous()
    assert got.tolist() == [expect]


def test_document_starts_is_monotone_and_bounded():
    g = torch.Generator().manual_seed(0)
    starts = torch.rand(4, 300, generator=g) < 0.05
    pos = data_utils.positions_from_starts(starts)
    ds = ops.document_starts(pos).long()
    idx = torch.arange(300)
    assert (ds[:, 1:] >= ds[:, :-1]).all() and (ds <= idx).all() and (ds[:, 0] == 0).all()
    assert ((ds == idx) == (pos == 0)).all()


# ---------------------------------------------------------------------------------------------------------------
# masked reference attention
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("nh,nkv", [(4, 4), (4, 2)])
def test_masked_reference_equals_per_document_attention(nh, nkv):
    g = torch.Generator().manual_seed(1)
    lengths = [5, 1, 17, 9]
    S = sum(lengths)
    q = torch.randn(2, S, nh, 16, generator=g, dtype=torch.float64)
    k = torch.randn(2, S, nkv, 16, generator=g, dtype=torch.float64)
    v = torch.randn(2, S, nkv, 16, generator=g, dtype=torch.float64)
    _, ds = _starts_from_lengths(lengths)
    o = ref.attention(q, k, v, doc_start=ds[None].expand(2, S))
    parts, a = [], 0
    for n in lengths:
        parts.append(ref.attention(q[:, a:a + n], k[:, a:a + n], v[:, a:a + n]))
        a += n
    torch.testing.assert_close(o, torch.cat(parts, dim=1), rtol=1e-5, atol=1e-6)   # fp32 softmax inside


def test_attention_qkv_cpu_path_honours_doc_start():
    g = torch.Generator().manual_seed(2)
    qkv = torch.randn(1, 12, 6, 8, generator=g)
    ds = ops.document_starts(torch.tensor([[0, 1, 2, 0, 1, 2, 3, 0, 1, 2, 3, 4]]))
    o = ops.attention_qkv(qkv, 2, 2, doc_start=ds)
    expect = ref.attention(qkv[:, :, :2], qkv[:, :, 2:4], qkv[:, :, 4:], doc_start=ds)
    torch.testing.assert_close(o, expect)
    # the first token of a document sees only itself: its output is its own v
    torch.testing.assert_close(o[0, 3], qkv[0, 3, 4:])


def test_cross_document_targets_are_dropped():
    _, ds = _starts_from_lengths([3, 2, 4])
    labels = torch.arange(10, 19)[None]
    tgt = ref.drop_cross_document_targets(ref.shift_labels(labels), ds[None])
    assert tgt.tolist() == [[11, 12, -100, 14, -100, 16, 17, 18, -100]]


# ---------------------------------------------------------------------------------------------------------------
# the model: a packed row against each document alone
# ---------------------------------------------------------------------------------------------------------------
def _fp32_llama():
    from distributed_training_guide_b200.models import get_config
    from distributed_training_guide_b200.models.llama import build_llama

    return build_llama(get_config("debug-llama"), dtype=torch.float32, device="cpu", seed=0)


@pytest.mark.parametrize("lengths", [[40], [7, 1, 20, 12], [1, 1, 30, 2, 6]])
def test_packed_row_matches_documents_alone(lengths):
    model = _fp32_llama()
    model.document_masking = True
    S = sum(lengths)
    g = torch.Generator().manual_seed(3)
    ids = torch.randint(0, model.config.vocab_size, (1, S), generator=g)
    pos, _ = _starts_from_lengths(lengths)
    with torch.no_grad():
        packed = model(ids, labels=ids, position_ids=pos[None], return_logits=True)
        a, loss_sum, n_tgt = 0, 0.0, 0
        for n in lengths:
            alone = model(ids[:, a:a + n], labels=ids[:, a:a + n], return_logits=True)
            torch.testing.assert_close(packed.logits[:, a:a + n], alone.logits, rtol=1e-5, atol=1e-5)
            loss_sum += float(alone.loss) * (n - 1)
            n_tgt += n - 1
            a += n
    if n_tgt:
        assert abs(float(packed.loss) - loss_sum / n_tgt) < 1e-5
    else:
        assert float(packed.loss) == 0.0


def test_flag_off_uses_position_ids_for_rope_only():
    model = _fp32_llama()
    ids = torch.randint(0, model.config.vocab_size, (1, 24), generator=torch.Generator().manual_seed(4))
    pos, _ = _starts_from_lengths([10, 14])
    with torch.no_grad():
        off = model(ids, labels=ids, position_ids=pos[None], return_logits=True)
        model.document_masking = True
        plain = model(ids, labels=ids, return_logits=True)
        model.document_masking = False
        ref_plain = model(ids, labels=ids, return_logits=True)
    # no position_ids: one document per row, as without the flag
    torch.testing.assert_close(plain.logits, ref_plain.logits, rtol=0, atol=0)
    assert float(plain.loss) == float(ref_plain.loss)
    # flag off: attention still crosses the boundary, so the second document's logits differ from masking
    model.document_masking = True
    with torch.no_grad():
        on = model(ids, labels=ids, position_ids=pos[None], return_logits=True)
    torch.testing.assert_close(off.logits[:, :10], on.logits[:, :10], rtol=1e-5, atol=1e-5)
    assert (off.logits[:, 10:] - on.logits[:, 10:]).abs().max() > 1e-3


def test_activation_checkpointing_passes_doc_start():
    model = _fp32_llama()
    model.document_masking = True
    ids = torch.randint(0, model.config.vocab_size, (2, 32), generator=torch.Generator().manual_seed(5))
    pos = data_utils.positions_from_starts(torch.tensor([[i in (0, 9, 20) for i in range(32)]] * 2))

    def grads(ckpt):
        model.zero_grad(set_to_none=True)
        model.activation_checkpointing = ckpt
        out = model(ids, labels=ids, position_ids=pos)
        out.loss.backward()
        return float(out.loss.detach()), {n: p.grad.clone() for n, p in model.named_parameters() if p.grad is not None}

    l0, g0 = grads(False)
    l1, g1 = grads(True)
    assert l0 == pytest.approx(l1, abs=1e-6)
    for n in g0:
        torch.testing.assert_close(g1[n], g0[n], rtol=1e-5, atol=1e-6)


# ---------------------------------------------------------------------------------------------------------------
# data sources
# ---------------------------------------------------------------------------------------------------------------
class _Args:
    def __init__(self, **kw):
        self.dataset_subset, self.model_name, self.seed, self.batch_size = None, "debug-llama", 0, 2
        self.num_samples, self.document_masking, self.eos_token_id = None, False, None
        self.__dict__.update(kw)


def _config():
    from distributed_training_guide_b200.models import get_config

    return get_config("debug-llama")


def _check_positions(pos):
    assert pos.dtype == torch.int64 and int(pos[0]) == 0
    ok = (pos[1:] == pos[:-1] + 1) | (pos[1:] == 0)
    assert bool(ok.all())


@pytest.mark.parametrize("kind", ["txt", "jsonl"])
def test_text_sources_make_each_text_a_document(tmp_path, kind):
    texts = ["alpha beta", "x", "a much longer line of text that spans a chunk boundary for sure", "tail"]
    path = tmp_path / f"d.{kind}"
    if kind == "txt":
        path.write_text("".join(t + "\n" for t in texts))
        lens = [len(t) + 2 for t in texts]       # bytes + newline + end-of-document id
    else:
        path.write_text("".join(json.dumps({"text": t}) + "\n" for t in texts))
        lens = [len(t) + 1 for t in texts]
    S = 16
    args = _Args(dataset_name=str(path), seq_length=S, document_masking=True)
    ds = data_utils.load_and_preprocess_data(args, _config())
    expect = torch.cat([torch.arange(n) for n in lens])
    for i in range(len(ds)):
        sample = ds[i]
        assert set(sample) == {"input_ids", "attention_mask", "labels", "position_ids"}
        chunk = expect[i * S:(i + 1) * S]
        want = data_utils.positions_from_starts(chunk == 0)   # a cut document restarts at 0
        assert sample["position_ids"].tolist() == want.tolist()
        _check_positions(sample["position_ids"])


def _write_bin(tmp_path, ids):
    path = tmp_path / "tokens.bin"
    np.asarray(ids, dtype=np.uint16).tofile(path)
    return str(path)


def test_bin_positions_after_eos(tmp_path):
    eos = 2
    ids = [5, 6, eos, 7, eos, eos, 8, 9, 10, 11, eos, 12, 13, 14, 15, 16]
    path = _write_bin(tmp_path, ids)
    args = _Args(dataset_name=path, seq_length=8, document_masking=True, eos_token_id=eos)
    ds = data_utils.load_and_preprocess_data(args, _config())
    assert ds[0]["position_ids"].tolist() == [0, 1, 2, 0, 1, 0, 0, 1]
    assert ds[1]["position_ids"].tolist() == [0, 1, 2, 0, 1, 2, 3, 4]
    # the loader that serves .bin files adds the same positions after the copy to the device
    dl = data_utils.build_dataloader(ds, batch_size=2, num_workers=0)
    for batch in dl:
        out = data_utils.to_device(batch, "cpu")
        assert torch.equal(out["position_ids"], data_utils.positions_after_eos(out["input_ids"], eos))
        for row in out["position_ids"]:
            _check_positions(row)


def test_bin_without_eos_is_refused_up_front(tmp_path):
    path = _write_bin(tmp_path, list(range(64)))
    with pytest.raises(ValueError, match="--eos-token-id"):
        data_utils.load_and_preprocess_data(_Args(dataset_name=path, seq_length=8, document_masking=True), _config())
    from distributed_training_guide_b200.trainer import run_chapter
    from distributed_training_guide_b200.parallel.strategies import SingleDevice

    with pytest.raises(ValueError, match="--eos-token-id"):   # before the model is built
        run_chapter("01-single-gpu", SingleDevice, ["-d", path, "-m", "debug-llama", "--document-masking", "--device",
                                                    "cpu"])


def test_synthetic_is_deterministic_and_keeps_its_tokens():
    plain = data_utils.SyntheticTokens(8, 64, 100, seed=3)
    a = data_utils.SyntheticTokens(8, 64, 100, seed=3, document_masking=True)
    b = data_utils.SyntheticTokens(8, 64, 100, seed=3, document_masking=True)
    c = data_utils.SyntheticTokens(8, 64, 100, seed=4, document_masking=True)
    assert torch.equal(a.tokens, plain.tokens)
    assert all(torch.equal(a[i]["position_ids"], b[i]["position_ids"]) for i in range(8))
    assert not all(torch.equal(a[i]["position_ids"], c[i]["position_ids"]) for i in range(8))
    n_docs = 0
    for i in range(8):
        p = a[i]["position_ids"]
        _check_positions(p)
        n_docs += int((p == 0).sum())
        assert int(p.max()) < 32   # document lengths are at most seq_length // 2
    assert n_docs > 8


@pytest.mark.parametrize("source", ["synthetic", "txt", "bin"])
def test_batch_keys_unchanged_without_the_flag(tmp_path, source):
    if source == "synthetic":
        name = "synthetic"
    elif source == "txt":
        name = str(tmp_path / "d.txt")
        (tmp_path / "d.txt").write_text("hello world\n" * 20)
    else:
        name = _write_bin(tmp_path, list(range(64)))
    ds = data_utils.load_and_preprocess_data(_Args(dataset_name=name, seq_length=8, eos_token_id=1), _config())
    assert set(ds[0]) == {"input_ids", "attention_mask", "labels"}
    dl = data_utils.build_dataloader(ds, batch_size=2, num_workers=0)
    batch = data_utils.to_device(next(iter(dl)), "cpu")
    assert set(batch) == {"input_ids", "attention_mask", "labels"}


# ---------------------------------------------------------------------------------------------------------------
# CLI and the engines that refuse the flag
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("chapter", ["01-single-gpu", "02-distributed-data-parallel", "04-fully-sharded-data-parallel",
                                     "05-training-llama-405b", "06-tensor-parallel", "07-2d-parallel", "deepspeed"])
def test_document_masking_flag_matrix(chapter):
    from distributed_training_guide_b200.utils.cli import get_parser

    base = ["-d", "synthetic", "-m", "debug-llama"]
    p = get_parser(chapter)
    assert p.parse_args(base).__dict__.get("document_masking", False) is False
    if chapter in ("01-single-gpu", "02-distributed-data-parallel", "04-fully-sharded-data-parallel",
                   "05-training-llama-405b"):
        a = p.parse_args(base + ["--document-masking", "--eos-token-id", "7"])
        assert a.document_masking is True and a.eos_token_id == 7
    else:
        with pytest.raises(SystemExit):
            p.parse_args(base + ["--document-masking"])


@pytest.mark.parametrize("parallelism", ["tp", "2d"])
def test_document_masking_rejected_by_tensor_parallel_engines(parallelism):
    from distributed_training_guide_b200.engine import TrainEngine

    with pytest.raises(ValueError, match="single, ddp, ddp_allreduce, fsdp"):
        TrainEngine.create("debug-llama", parallelism=parallelism, device="cpu", document_masking=True)


def test_document_masking_rejected_for_gpt2():
    from distributed_training_guide_b200.engine import TrainEngine

    with pytest.raises(ValueError, match="Llama"):
        TrainEngine.create("debug-gpt2", parallelism="single", device="cpu", document_masking=True)


def test_chapter_01_trains_with_document_masking(tmp_path):
    from distributed_training_guide_b200.parallel.strategies import SingleDevice
    from distributed_training_guide_b200.trainer import run_chapter

    state, info = run_chapter("01-single-gpu", SingleDevice,
                              ["-d", "synthetic", "-m", "debug-llama", "--document-masking", "--device", "cpu",
                               "-s", "64", "-b", "2", "--max-steps", "3", "--log-freq", "1", "--num-workers", "0",
                               "--save-dir", str(tmp_path)])
    assert state["global_step"] == 3 and np.isfinite(info["running_loss"])


# ---------------------------------------------------------------------------------------------------------------
# DDP and FSDP over gloo against one process
# ---------------------------------------------------------------------------------------------------------------
_CUTS = (0, 5, 6, 19, 27)


def _packed_batch(vocab, seed, rank, B=2, S=32):
    g = torch.Generator().manual_seed(1000 * seed + rank)
    ids = torch.randint(0, vocab, (B, S), generator=g)
    pos = data_utils.positions_from_starts(torch.tensor([[i in _CUTS for i in range(S)]] * B))
    return {"input_ids": ids, "labels": ids.clone(), "position_ids": pos}


def _train_dist(rank, world, parallelism, steps):
    from distributed_training_guide_b200.engine import TrainEngine

    torch.manual_seed(0)
    eng = TrainEngine.create("debug-llama", parallelism=parallelism, batch_size=2, seq_length=32, device="cpu",
                             lr=1e-3, document_masking=True)
    assert eng.model.document_masking
    losses = [float(eng.step(_packed_batch(eng.config.vocab_size, i, eng.strategy.dp_rank))) for i in range(steps)]
    if parallelism == "fsdp":
        sd = eng.strategy.engine.full_state_dict()
    else:
        sd = eng.model.state_dict()
    return losses, {k: v.detach().float().clone() for k, v in sd.items()}


@pytest.mark.parametrize("parallelism", ["ddp", "fsdp"])
def test_distributed_document_masking_matches_single_process(parallelism):
    from distributed_training_guide_b200.engine import TrainEngine

    steps, world = 3, 2
    (l0, sd0), (l1, sd1) = run_distributed(_train_dist, world=world, args=(parallelism, steps))
    torch.manual_seed(0)
    eng = TrainEngine.create("debug-llama", parallelism="single", batch_size=2 * world, seq_length=32, device="cpu",
                             lr=1e-3, document_masking=True)
    ref_losses = []
    for i in range(steps):
        parts = [_packed_batch(eng.config.vocab_size, i, r) for r in range(world)]
        batch = {k: torch.cat([p[k] for p in parts]) for k in parts[0]}
        ref_losses.append(float(eng.step(batch)))
    ref_sd = {k: v.detach().float() for k, v in eng.model.state_dict().items()}
    # every rank has the same number of targets, so the mean of the rank losses is the global loss
    for i in range(steps):
        assert abs(0.5 * (l0[i] + l1[i]) - ref_losses[i]) < 2e-2, (i, l0[i], l1[i], ref_losses[i])
    for k in sd0:
        assert np.array_equal(sd0[k], sd1[k]), k   # results come back from the workers as numpy arrays
        assert np.abs(sd0[k] - ref_sd[k].numpy()).max() < 2e-2, k
