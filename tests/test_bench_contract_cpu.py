"""bench.py end to end on the CPU (debug model, CUDA timing primitives replaced by stand-ins): the JSON line the driver
parses must carry every key of the contract, whatever happened to the code around it."""
import contextlib
import io
import json
import sys
from pathlib import Path
from types import SimpleNamespace
from unittest import mock

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))


class _Ev:
    _t = 0.0

    def __init__(self, *a, **k):
        self.t = None

    def record(self, *a):
        import time

        self.t = time.perf_counter()

    def synchronize(self):
        pass

    def elapsed_time(self, other):
        return 1000.0 * ((other.t or 0.0) - (self.t or 0.0))


def test_bench_prints_the_contract_json(capsys):
    import bench

    args = SimpleNamespace(gpus=1, steps=2, warmup=3, impl="b200", model="debug-llama", seq_len=64, batch=2,
                           parallelism="ddp", tensor_parallel=None, layers=None, dump_outputs=None)
    patches = [mock.patch("torch.cuda.Event", _Ev), mock.patch("torch.cuda.synchronize", lambda *a, **k: None),
               mock.patch("torch.cuda.max_memory_allocated", lambda *a, **k: 0),
               mock.patch.dict("os.environ", {"DTG_PHASE_TIMING": "1", "WORLD_SIZE": "1"})]
    with contextlib.ExitStack() as es:
        for p in patches:
            es.enter_context(p)
        bench.run_b200(args)
    import faulthandler

    faulthandler.cancel_dump_traceback_later()
    out = capsys.readouterr().out.strip().splitlines()
    line = json.loads(out[-1])
    for key in ("metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling",
                "vs_baseline", "dtype", "data", "config", "clocks", "e2e", "gpu_launches"):
        assert key in line, key
    assert line["unit"] == "tokens/s" and line["n_gpus"] == 1 and line["steps"] == 2 and line["warmup"] == 3
    assert line["higher_is_better"] is True and line["scaling"] == "weak" and line["dtype"] == "bf16"
    assert set(line["config"]) >= {"model", "global_batch", "seq_len", "parallelism"}
    assert set(line["e2e"]) >= {"value", "unit", "h2d_bytes_per_step", "d2h_bytes_per_step"}
    assert line["e2e"]["h2d_bytes_per_step"] == 3 * 2 * 64 * 8 and line["e2e"]["d2h_bytes_per_step"] == 4
    assert set(line["clocks"]) >= {"sm_mhz", "sm_max_mhz", "reasons"}
    assert line["value"] > 0 and line["ms_per_step"] > 0 and line["config"]["global_batch"] == 2
    assert abs(line["value"] - 1000.0 * 2 * 64 / line["ms_per_step"]) < 1e-6 * line["value"]


def _bench_dump(out_dir, steps):
    import bench

    args = SimpleNamespace(gpus=1, steps=steps, warmup=1, impl="b200", model="debug-llama", seq_len=64, batch=1,
                           parallelism="ddp", tensor_parallel=None, layers=None, dump_outputs=str(out_dir))
    with contextlib.ExitStack() as es:
        for p in [mock.patch("torch.cuda.Event", _Ev), mock.patch("torch.cuda.synchronize", lambda *a, **k: None),
                  mock.patch("torch.cuda.max_memory_allocated", lambda *a, **k: 0),
                  mock.patch.dict("os.environ", {"WORLD_SIZE": "1"})]:
            es.enter_context(p)
        with contextlib.redirect_stdout(io.StringIO()) as buf:
            bench.run_b200(args)
    import faulthandler

    faulthandler.cancel_dump_traceback_later()
    return json.loads([l for l in buf.getvalue().splitlines() if l.startswith("{")][-1])


def test_bench_dump_outputs_is_reproducible(tmp_path):
    """--dump-outputs: the last timed step's loss and a seeded weight sample, float32, identical for identical
    arguments, and different when --steps changes how many timed steps ran."""
    import numpy as np

    a = _bench_dump(tmp_path / "a", steps=2)
    _bench_dump(tmp_path / "b", steps=2)
    c = _bench_dump(tmp_path / "c", steps=3)
    assert a["steps"] == 2 and c["steps"] == 3
    for name in ("loss.npy", "params_sample.npy"):
        x, y = np.load(tmp_path / "a" / name), np.load(tmp_path / "b" / name)
        assert x.dtype == np.float32 and x.size > 0 and (tmp_path / "a" / name).stat().st_size < 64 << 20
        assert np.array_equal(x, y), name
    assert not np.array_equal(np.load(tmp_path / "a" / "params_sample.npy"), np.load(tmp_path / "c" / "params_sample.npy"))


def _bench_rank(rank, world):
    import io

    import bench

    args = SimpleNamespace(gpus=world, steps=2, warmup=3, impl="b200", model="debug-llama", seq_len=64, batch=1,
                           parallelism="ddp", tensor_parallel=None, layers=None, dump_outputs=None)
    buf = io.StringIO()
    with contextlib.ExitStack() as es:
        for p in [mock.patch("torch.cuda.Event", _Ev), mock.patch("torch.cuda.synchronize", lambda *a, **k: None),
                  mock.patch("torch.cuda.max_memory_allocated", lambda *a, **k: 0)]:
            es.enter_context(p)
        with contextlib.redirect_stdout(buf):
            bench.run_b200(args)
    import faulthandler

    faulthandler.cancel_dump_traceback_later()
    lines = [l for l in buf.getvalue().splitlines() if l.startswith("{")]
    return lines[-1] if lines else ""


def test_bench_two_ranks_prints_one_line_with_whole_job_tokens():
    from dist_utils import run_distributed

    r0, r1 = run_distributed(_bench_rank, world=2, timeout=300)
    assert r1 == ""                                   # only rank 0 prints
    line = json.loads(r0)
    assert line["n_gpus"] == 2 and line["config"]["global_batch"] == 2 and "dp2" in line["config"]["parallelism"]
    assert abs(line["value"] - 1000.0 * 2 * 64 / line["ms_per_step"]) < 1e-6 * line["value"]   # whole-job aggregate
    assert "exposed_comm_ms" in line
