"""Qwen3-MoE benchmark on one GPU (Qwen3-30B-A3B's shapes by default: 128 experts, top-8, H 2048, expert I 768, S 4096,
B 1): prints one JSON record with the card's name and power limit.

  * all six grouped GEMMs of a training step (forward gate|up and down, dgrad of both, wgrad of both): useful TFLOP/s
    over the real rows only, and the share of permuted rows that are 128-row segment padding;
  * GB/s of route (raw and renormalised weights), permute and combine;
  * device-timed tokens/s and peak memory of single-GPU training steps of the model truncated to ``--layers`` layers
    (the whole model does not fit one GPU).

The timing helpers and the training loop are ``bench_olmoe``'s.

    python bench_qwen3_moe.py [--model Qwen/Qwen3-30B-A3B] [--seq 4096] [--layers 4] [--steps 3] [--warmup 1]
"""
import argparse
import json
import sys

import torch

from bench_olmoe import _card, _time, steps


def kernels(T, E, k, H, I):
    from distributed_training_guide_b200 import _ext

    C = _ext.load(required=True)
    bf = dict(device="cuda", dtype=torch.bfloat16)
    g = torch.Generator(device="cuda").manual_seed(0)
    lg = torch.randn(T, E, device="cuda", generator=g).to(torch.bfloat16)
    x = torch.randn(T, H, device="cuda", generator=g).to(torch.bfloat16)
    gate_up = (torch.randn(E, 2 * I, H, device="cuda", generator=g) * 0.02).to(torch.bfloat16)
    down = (torch.randn(E, H, I, device="cuda", generator=g) * 0.02).to(torch.bfloat16)
    p, idx, w, pos, seg, tiles, row_tok, counts = C.moe_route(lg, k, True)
    xp = C.moe_permute(x, row_tok, seg, k)
    R = xp.shape[0]
    used = seg[-1].item()
    gu = torch.randn(R, 2 * I, device="cuda", generator=g).to(torch.bfloat16)
    h = torch.randn(R, I, device="cuda", generator=g).to(torch.bfloat16)
    yp = torch.empty(R, H, **bf)
    dyp = torch.randn(R, H, device="cuda", generator=g).to(torch.bfloat16)
    dh, dxp = torch.empty(R, I, **bf), torch.empty(R, H, **bf)
    d_gate_up, d_down = torch.empty_like(gate_up), torch.empty_like(down)
    real = T * k
    gemms = {   # name: (launch, useful FLOPs over the real rows)
        "fwd_gate_up": (lambda: C.gemm_grouped(0, xp, gate_up, gu, seg, tiles), 2.0 * real * 2 * I * H),
        "fwd_down": (lambda: C.gemm_grouped(0, h, down, yp, seg, tiles), 2.0 * real * H * I),
        "dgrad_down": (lambda: C.gemm_grouped(1, dyp, down, dh, seg, tiles), 2.0 * real * I * H),
        "dgrad_gate_up": (lambda: C.gemm_grouped(1, gu, gate_up, dxp, seg, tiles), 2.0 * real * H * 2 * I),
        "wgrad_down": (lambda: C.gemm_grouped(2, dyp, h, d_down, seg), 2.0 * real * H * I),
        "wgrad_gate_up": (lambda: C.gemm_grouped(2, gu, xp, d_gate_up, seg), 2.0 * real * 2 * I * H),
    }
    out = {"tokens": T, "experts": E, "top_k": k, "H": H, "I": I, "permuted_rows": used,
           "padding_share": round(1 - real / used, 4)}
    total_t = total_f = 0.0
    for name, (fn, flop) in gemms.items():
        t = _time(fn)
        total_t += t
        total_f += flop
        out[f"{name}_us"] = round(t * 1e6, 1)
        out[f"{name}_tflops"] = round(flop / t / 1e12, 1)
    out["six_gemms_tflops"] = round(total_f / total_t / 1e12, 1)
    route_bytes = T * E * 2 + T * E * 4 + T * k * 16 + R * 4
    for norm in (False, True):
        t = _time(lambda: C.moe_route(lg, k, norm))
        tag = "route_norm" if norm else "route_raw"
        out[f"{tag}_us"], out[f"{tag}_gbps"] = round(t * 1e6, 1), round(route_bytes / t / 1e9, 1)
    t = _time(lambda: C.moe_permute(x, row_tok, seg, k))
    out["permute_us"], out["permute_gbps"] = round(t * 1e6, 1), round((T * H + used * H) * 2 / t / 1e9, 1)
    t = _time(lambda: C.moe_combine(yp, pos, w))
    out["combine_us"] = round(t * 1e6, 1)
    out["combine_gbps"] = round(((T * k * H + T * H) * 2 + T * k * 8) / t / 1e9, 1)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="Qwen/Qwen3-30B-A3B")
    ap.add_argument("--seq", type=int, default=4096)
    ap.add_argument("--layers", type=int, default=4, help="train only the first N layers (0: skip training)")
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_qwen3_moe.py measures on a GPU; none is visible")
    from distributed_training_guide_b200.models.configs import get_config

    cfg = get_config(a.model)
    rec = {"card": _card(), "kernels": kernels(a.seq, cfg.num_experts, cfg.num_experts_per_tok, cfg.hidden_size,
                                               cfg.intermediate_size)}
    if a.layers:
        try:
            rec["train"] = steps(a.model, a.seq, a.steps, a.warmup, a.layers)
        except torch.OutOfMemoryError as e:
            rec["train"] = {"model": a.model, "layers": a.layers, "error": f"out of memory: {str(e).splitlines()[0]}"}
    print(json.dumps(rec))


if __name__ == "__main__":
    main()
