#!/usr/bin/env python3
"""Cluster-wide GPU monitor: polls every host in a hosts file with ``nvidia-smi`` over ssh and prints
per-node and cluster averages of utilisation, power (% of limit), memory (% used) and the number of
compute processes.  A hung NCCL / NVLink-barrier job shows up as ~10 % power with 100 % "utilisation",
a dead worker as a drop in the process count (see diagnosing-errors/README.md).

    python top-cluster.py hosts [--poll-freq 1000] [--once] [--local]

Same purpose and CLI as the reference's top-cluster.py.
"""
import argparse
import concurrent.futures as cf
import subprocess
import sys
import time

QUERY = "utilization.gpu,power.draw,power.limit,memory.used,memory.total"


def _run(cmd, timeout):
    try:
        return subprocess.run(cmd, capture_output=True, text=True, timeout=timeout).stdout
    except Exception:
        return ""


def probe(host, local=False, timeout=15.0):
    base = [] if local else ["ssh", "-o", "BatchMode=yes", "-o", "ConnectTimeout=5", host]
    gpus = _run(base + ["nvidia-smi", f"--query-gpu={QUERY}", "--format=csv,noheader,nounits"], timeout)
    apps = _run(base + ["nvidia-smi", "--query-compute-apps=pid", "--format=csv,noheader"], timeout)
    rows = []
    for line in gpus.strip().splitlines():
        try:
            rows.append([float(x) for x in line.split(",")])
        except ValueError:
            pass
    if not rows:
        return {"host": host, "ok": False}
    n = len(rows)
    return {
        "host": host, "ok": True, "gpus": n,
        "util": sum(r[0] for r in rows) / n,
        "power": 100.0 * sum(r[1] / max(r[2], 1.0) for r in rows) / n,
        "mem": 100.0 * sum(r[3] / max(r[4], 1.0) for r in rows) / n,
        "procs": len([p for p in apps.strip().splitlines() if p.strip()]),
    }


def render(stats):
    lines = [f"{'host':<24}{'gpus':>5}{'util %':>9}{'power %':>9}{'mem %':>8}{'procs':>7}"]
    good = [s for s in stats if s["ok"]]
    for s in stats:
        if s["ok"]:
            lines.append(f"{s['host']:<24}{s['gpus']:>5}{s['util']:>9.1f}{s['power']:>9.1f}{s['mem']:>8.1f}{s['procs']:>7}")
        else:
            lines.append(f"{s['host']:<24}  unreachable")
    if good:
        k = len(good)
        lines.append("-" * 62)
        lines.append(f"{'cluster (' + str(k) + ' nodes)':<24}{sum(s['gpus'] for s in good):>5}"
                     f"{sum(s['util'] for s in good) / k:>9.1f}{sum(s['power'] for s in good) / k:>9.1f}"
                     f"{sum(s['mem'] for s in good) / k:>8.1f}{sum(s['procs'] for s in good):>7}")
    return "\n".join(lines)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("hosts", help="file with one hostname per line")
    ap.add_argument("--poll-freq", type=int, default=1000, help="milliseconds between polls")
    ap.add_argument("--once", action="store_true")
    ap.add_argument("--local", action="store_true", help="treat every host as this machine (no ssh)")
    args = ap.parse_args()
    with open(args.hosts) as fp:
        hosts = [h.strip() for h in fp if h.strip() and not h.startswith("#")]
    with cf.ThreadPoolExecutor(max_workers=max(4, len(hosts))) as ex:
        while True:
            stats = list(ex.map(lambda h: probe(h, args.local), hosts))
            print(("" if args.once else "\033[2J\033[H") + time.strftime("%H:%M:%S") + "\n" + render(stats), flush=True)
            if args.once:
                return 0 if all(s["ok"] for s in stats) else 1
            time.sleep(args.poll_freq / 1000.0)


if __name__ == "__main__":
    sys.exit(main())
