"""Operational tools: the cluster monitor (against a fake nvidia-smi) and the pre-download helper's offline path."""
import os
import stat
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent

FAKE_SMI = """#!/bin/bash
if [[ "$*" == *query-gpu* ]]; then
  for i in 0 1 2 3; do echo "100, 985.2, 1000.0, 129000, 183359"; done
else
  for i in 0 1 2 3; do echo "$((4000 + i))"; done
fi
"""


def test_top_cluster_renders_nodes_and_cluster_average(tmp_path):
    smi = tmp_path / "nvidia-smi"
    smi.write_text(FAKE_SMI)
    smi.chmod(smi.stat().st_mode | stat.S_IEXEC)
    hosts = tmp_path / "hosts"
    hosts.write_text("node-a\n# a comment\nnode-b\n")
    env = dict(os.environ, PATH=f"{tmp_path}:{os.environ['PATH']}")
    r = subprocess.run([sys.executable, str(ROOT / "top-cluster.py"), str(hosts), "--once", "--local"],
                       capture_output=True, text=True, env=env, timeout=60)
    assert r.returncode == 0, r.stderr
    lines = [l for l in r.stdout.splitlines() if l.strip()]
    assert any(l.startswith("node-a") for l in lines) and any(l.startswith("node-b") for l in lines)
    node = next(l for l in lines if l.startswith("node-a")).split()
    assert node[1] == "4" and abs(float(node[2]) - 100.0) < 1e-6            # gpus, util %
    assert abs(float(node[3]) - 98.5) < 0.1 and abs(float(node[4]) - 70.4) < 0.1   # power %, mem %
    assert node[5] == "4"                                                   # compute processes
    total = next(l for l in lines if l.startswith("cluster (2 nodes)")).split()
    assert total[-1] == "8" and total[3] == "8"


def test_download_helper_falls_back_to_embedded_config():
    env = dict(os.environ, HF_HUB_OFFLINE="1", TRANSFORMERS_OFFLINE="1")
    r = subprocess.run([sys.executable, str(ROOT / "05-training-llama-405b" / "download.py"), "-m",
                        "meta-llama/Llama-3.1-405B", "--skip-model"], capture_output=True, text=True, env=env, timeout=300)
    assert r.returncode == 0, r.stderr
    assert "405.85 B parameters" in r.stdout or "cached" in r.stdout, r.stdout


def test_bench_watchdog_dumps_stacks_and_exits():
    """bench.py arms a watchdog per stage: a stage that stalls past its budget dumps every thread's stack and exits
    instead of hanging until the caller's limit."""
    code = ("import sys, time; sys.path.insert(0, %r); import bench; bench._stage('stalling stage', budget_s=1); "
            "time.sleep(30)") % str(ROOT)
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=60)
    assert r.returncode == 3
    assert "stalling stage" in r.stderr and "WATCHDOG" in r.stderr and "most recent call first" in r.stderr  # the stack dump


def test_bench_stage_budgets_fit_the_driver_limit():
    """The sum of every stage budget at the driver's configuration (20 steps / 5 warm-up) stays below its
    870 s per-N limit: a wedged run must diagnose itself, never be killed silently from outside."""
    sys.path.insert(0, str(ROOT))
    import bench

    total = sum(bench.BUDGET.values()) + 2 * 5 + 2 * 2 * 20
    assert total < 870, total


def test_both_bench_arms_describe_the_same_config():
    """The driver compares the two arms' ``config`` dicts: same model / batch / sequence / mesh strings from one helper."""
    from types import SimpleNamespace

    sys.path.insert(0, str(ROOT))
    import bench

    a = SimpleNamespace(model="meta-llama/Llama-2-7b-hf", layers=None, batch=1, seq_len=4096)
    own = bench._config(a, 8, 1, "ddp")
    ref = bench._config(a, 8, 1, "ddp")
    assert own == ref and own["parallelism"] == "dp8 (ddp+zero1)" and own["global_batch"] == 8 and "l2" in own
    assert bench._config(a, 2, 4, "2d")["parallelism"] == "dp2xtp4 (fsdp x tp)"
