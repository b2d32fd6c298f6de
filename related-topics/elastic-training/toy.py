"""Fault-injection toy for elastic restarts (no GPU needed).

    torchrun --standalone --local-addr 127.0.0.1 --nproc-per-node 4 --max-restarts 3 toy.py

Every rank "trains" by sleeping; each step a rank fails with a small probability.  torchrun then
tears the whole gang down and restarts it, and the job resumes from the step recorded in
``toy-state.json`` — the same state-file resume protocol the chapter scripts use (``state.json``).
``@record`` writes the failing rank's traceback to $TORCHELASTIC_ERROR_FILE.
"""
import argparse
import json
import os
import random
import time

import torch.distributed as dist
from torch.distributed.elastic.multiprocessing.errors import record

STATE = os.environ.get("TOY_STATE_FILE", "./toy-state.json")


def init_process_group(timeout):
    """gloo process group of this attempt, with its store keys under a per-attempt prefix.

    torchrun hands its workers the TCPStore of its own rendezvous and keeps that store across restarts, so the
    keys a failed attempt wrote (among them the listening address of every gloo peer) are still there when the
    restarted gang sets up.  A worker can then read a dead peer's address and fail to connect ("Connection
    refused"; the next attempt may hang on a stale counter instead), which burns the restarts.  Prefixing every
    key with the restart count gives each attempt a clean namespace."""
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    # without the shared store (TORCH_DISABLE_SHARE_RDZV_TCP_STORE=1) rank 0 hosts a fresh store per attempt
    hosted_by_agent = os.environ.get("TORCHELASTIC_USE_AGENT_STORE") == "True"
    store = dist.TCPStore(os.environ["MASTER_ADDR"], int(os.environ["MASTER_PORT"]), world,
                          is_master=not hosted_by_agent and rank == 0, timeout=timeout)
    store = dist.PrefixStore(f"toy/attempt_{os.environ.get('TORCHELASTIC_RESTART_COUNT', '0')}", store)
    dist.init_process_group(backend="gloo", store=store, rank=rank, world_size=world, timeout=timeout)


@record
def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=500)
    ap.add_argument("--failure-prob", type=float, default=0.001)
    ap.add_argument("--step-time", type=float, default=0.01)
    ap.add_argument("--fail-at-steps", type=int, nargs="*", default=[],
                    help="deterministic injection: fail once at each of these steps (besides the random failures)")
    args = ap.parse_args()

    import datetime

    init_process_group(datetime.timedelta(seconds=120))
    rank, world = dist.get_rank(), dist.get_world_size()
    state = {"num_steps": 0}
    if os.path.exists(STATE):
        with open(STATE) as fp:
            state = json.load(fp)
    if rank == 0:
        print(f"[restart count={os.environ.get('TORCHELASTIC_RESTART_COUNT', '0')}] world={world} "
              f"resuming at step {state['num_steps']}", flush=True)
    # different failure pattern after every restart, reproducible for a given (rank, world, step)
    random.seed(rank + world * state["num_steps"])
    while state["num_steps"] < args.steps:
        time.sleep(args.step_time)
        planned = state["num_steps"] in args.fail_at_steps and state["num_steps"] not in state.get("failed_at", [])
        if planned:
            if rank == 0:  # remember it, so the restarted gang passes this step
                state.setdefault("failed_at", []).append(state["num_steps"])
                with open(STATE, "w") as fp:
                    json.dump(state, fp)
            dist.barrier()
        if (planned and rank == state["num_steps"] % world) or random.random() < args.failure_prob:
            raise ValueError(f"injected failure on rank {rank} at step {state['num_steps']}")
        state["num_steps"] += 1
        dist.barrier()
        if rank == 0:
            tmp = STATE + ".tmp"
            with open(tmp, "w") as fp:
                json.dump(state, fp)
            os.replace(tmp, STATE)
        dist.barrier()
    if rank == 0:
        print(f"finished {state['num_steps']} steps", flush=True)
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
