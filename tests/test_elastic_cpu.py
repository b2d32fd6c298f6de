"""The elastic toy under torchrun: state-file resume across launches, and an injected failure followed by a
gang restart."""
import json
import os
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
TOY = str(ROOT / "related-topics" / "elastic-training" / "toy.py")


def _launch(tmp_path, extra, timeout):
    env = dict(os.environ, TOY_STATE_FILE=str(tmp_path / "toy-state.json"),
               TORCHELASTIC_ERROR_FILE=str(tmp_path / "error.json"))
    cmd = [sys.executable, "-m", "torch.distributed.run", "--standalone", "--local-addr", "127.0.0.1",
           "--nproc-per-node", "2", "--max-restarts", "3", "--monitor-interval", "1", TOY, "--failure-prob", "0.0",
           "--step-time", "0.001"] + extra
    return subprocess.run(cmd, capture_output=True, text=True, env=env, timeout=timeout)


def test_toy_resumes_from_state_file(tmp_path):
    r = _launch(tmp_path, ["--steps", "10"], 300)
    assert r.returncode == 0, (r.stdout + r.stderr)[-2000:]
    assert json.loads((tmp_path / "toy-state.json").read_text())["num_steps"] == 10
    r = _launch(tmp_path, ["--steps", "25"], 300)
    out = r.stdout + r.stderr
    assert r.returncode == 0, out[-2000:]
    assert "resuming at step 10" in out and "finished 25 steps" in out


def test_toy_injected_failure_restarts(tmp_path):
    """One restart must be enough: the restarted gang sets up its process group in a store namespace of its own, so
    no worker reads an address or counter the failed attempt left behind (which failed or hung about one run in
    three before)."""
    r = _launch(tmp_path, ["--steps", "20", "--fail-at-steps", "7"], 300)
    out = r.stdout + r.stderr
    assert r.returncode == 0, out[-2000:]
    assert "injected failure" in out and "resuming at step 7" in out and "finished 20 steps" in out
    assert "restart count=1" in out and "restart count=2" not in out, out[-2000:]
