"""Phases of one multifrontal linear solve on the bench's headline workload (config C5, pose graph of 2 500 SE3 poses, batch 2048), timed
with CUDA events after a warm-up, each over --reps calls:

  factor           Gram + numeric factorisation (thb_front_factor_f64), what bench.py reports as numeric_factorisation
  factor_forward   Gram + factorisation with the fused forward substitution of A^T b (thb_front_factor_forward_f64)
  forward          the forward substitution alone (thb_front_forward_f64)
  backward         the backward substitution alone (thb_front_backward_f64)
  substitute       both substitutions (thb_front_solve_f64), what bench.py reports as substitutions

factor_forward - factor is what the fused elimination costs inside the factor kernel; the solve of the fused path is factor_forward +
backward, that of the two-pass path factor + substitute.  Phases whose entry point the library does not export are reported as null.
The GPU's name and power limit are printed with the numbers.

    python tools/front_solve_phases.py [--batch 2048] [--reps 5] [--json OUT]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gpu_description():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()
        name, plim = (s.strip() for s in out[0].split(","))
        return name, plim
    except Exception:
        import torch
        return torch.cuda.get_device_name(), None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=2048)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--json", help="also write the result line to this file")
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "front_solve_phases.py needs a CUDA device"
    import theseus_b200 as th
    from theseus_b200 import _lib
    from theseus_b200.datasets import build_pose_graph_objective, pose_graph_sphere
    from theseus_b200.optimizer import convert_to_alpha_beta_damping_tensors
    from bench import C5_PER_RING, C5_RINGS

    device = torch.device("cuda", 0)
    torch.cuda.set_device(device)
    B = args.batch
    data = pose_graph_sphere(C5_RINGS, C5_PER_RING, B, seed=1000, device=device)
    objective, _ = build_pose_graph_objective(th, data, device)
    opt = th.LevenbergMarquardt(objective, linear_solver_cls=th.BaspachoSparseSolver, linearization_cls=th.SparseLinearization,
                                max_iterations=1, linear_solver_kwargs=dict(layout="front"))
    solver, lin = opt.linear_solver, opt.linear_solver.linearization
    with torch.no_grad():
        lin.linearize()
    A64, b64 = lin.A_val.detach().double().contiguous(), lin.b.detach().double().contiguous()
    lam = torch.full((B,), 1e-3, dtype=torch.float64, device=device)
    alpha, beta = convert_to_alpha_beta_damping_tensors(lam, 1e-8, True, B, device, torch.float64)
    lib = _lib.load()
    Atb = solver._numeric(A64, b64, alpha, beta)
    d = solver._dev
    bufs, L = d["bufs"], d["launches"]
    chunk = bufs["chunk"]

    def has(sym):
        try:
            getattr(lib, sym)
            return sym in _lib.SIGNATURES
        except AttributeError:
            return False

    def forward():
        for c0 in range(0, B, chunk):
            _lib.check(lib.thb_front_forward_f64(C.byref(d["front"]), L.ctypes.data, L.shape[0], _lib.ptr(bufs["factor"][c0:]), _lib.ptr(Atb[c0:]),
                                                 _lib.ptr(bufs["work"][c0:]), _lib.ptr(bufs["varena"]), min(chunk, B - c0), _lib.stream_ptr()),
                       "front_forward")

    phases = {"factor": lambda: solver._numeric(A64, b64, alpha, beta)}
    if has("thb_front_factor_forward_f64"):
        phases["factor_forward"] = lambda: solver._numeric_front(A64, b64, alpha, beta, forward=True)
    if has("thb_front_forward_f64"):
        phases["forward"] = forward
    if has("thb_front_backward_f64"):
        phases["backward"] = solver._backward_front
    phases["substitute"] = lambda: solver._substitute(Atb)

    def timed(fn):
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(args.reps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / args.reps

    with torch.no_grad():
        for fn in phases.values():   # warm-up: module loads, shared-memory opt-ins, allocator
            fn()
            fn()
        ms = {k: timed(fn) for k, fn in phases.items()}
    for k in ("factor_forward", "forward", "backward"):
        ms.setdefault(k, None)
    name, plim = gpu_description()
    line = dict(gpu=name, power_limit=plim, batch=B, chunk=chunk, reps=args.reps, ms_per_call=ms,
                fused_forward_cost_ms=(ms["factor_forward"] - ms["factor"]) if ms["factor_forward"] is not None else None,
                solve_two_pass_ms=ms["factor"] + ms["substitute"],
                solve_fused_ms=(ms["factor_forward"] + ms["backward"]) if ms["factor_forward"] is not None else None,
                launches_per_chunk=int(L.shape[0]))
    print(json.dumps(line))
    if args.json:
        with open(args.json, "w") as f:
            f.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()
