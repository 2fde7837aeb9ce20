"""Where the time of the dense-path fronts goes, kernel by kernel, on the bench's headline workload (config C5, pose graph of 2 500 SE3
poses, batch 2048, one linearization, damping 1e-3; at C5 the only such front is the 462-pivot root).

Like tools/front_launch_times.py, the launch rows of the dense-path fronts are called one at a time on one chunk of the batch, after the
rows before them ran once (so the children's update matrices are in the arena); here under torch.profiler with CUDA activities, in a run
of its own, with and without the fused forward substitution (--reps passes after two warm-up passes).  Prints ms per pass of every kernel
of those calls -- front_assemble_kernel / chol_col_kernel / front_extract_kernel / front_forward_kernel for the assembled form, or
chol_col_kernel / front_forward_kernel for the direct one -- with the GPU's name and power limit.  THB_FRONT_BIG_DIRECT=0 selects the
assembled form, THB_CHOL_GROUP (or --groups, one measurement per value) the ticket group size.  Needs a CUDA device.

    python tools/front_root_phases.py [--batch 2048] [--reps 10] [--groups 0,128,256] [--json OUT]
"""
import argparse
import ctypes as C
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=2048)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--groups", help="comma-separated THB_CHOL_GROUP values, one measurement each (0: the library's default)")
    ap.add_argument("--json", help="also write the result line to this file")
    args = ap.parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile
    assert torch.cuda.is_available(), "front_root_phases.py needs a CUDA device"
    import theseus_b200 as th
    from theseus_b200 import _lib
    from theseus_b200.datasets import build_pose_graph_objective, pose_graph_sphere
    from theseus_b200.optimizer import convert_to_alpha_beta_damping_tensors
    from bench import C5_PER_RING, C5_RINGS
    from front_solve_phases import gpu_description

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
    Atb = solver._numeric_front(A64, b64, alpha, beta, forward=True)
    d = solver._dev
    bufs, L = d["bufs"], d["launches"]
    nb, s = bufs["chunk"], _lib.stream_ptr()
    cols = L.shape[1]
    head = (_lib.ptr(bufs["factor"]), _lib.ptr(bufs["ata"]), solver._ata_size, _lib.ptr(alpha), _lib.ptr(beta), _lib.ptr(bufs["arena"]),
            _lib.ptr(bufs["ws"]) if d["max_np"] else None, bufs["ws"].numel(), _lib.ptr(bufs["info"]))
    fwd = (_lib.ptr(Atb), _lib.ptr(bufs["work"]), _lib.ptr(bufs["varena"]))

    def call(first, count, forward):
        rows = L.ctypes.data + first * cols * 8
        if forward:
            _lib.check(lib.thb_front_factor_forward_f64(C.byref(d["front"]), rows, count, *head, *fwd, nb, s), "front_factor_forward")
        else:
            _lib.check(lib.thb_front_factor_f64(C.byref(d["front"]), rows, count, *head, nb, s), "front_factor")

    dense = [q for q in range(L.shape[0]) if int(L[q, 1]) == 3]
    assert dense, "no dense-path front in the plan"
    call(0, dense[0], True)   # everything before the first dense-path front: its children's update matrices and border vectors

    def measure():
        out = {}
        for key, forward in (("factor", False), ("factor_forward", True)):
            for _ in range(2):
                for q in dense:
                    call(q, 1, forward)
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(args.reps):
                    for q in dense:
                        call(q, 1, forward)
                torch.cuda.synchronize()
            per = {}
            for ev in prof.key_averages():
                if ev.device_type == torch.autograd.DeviceType.CUDA and ev.self_device_time_total > 0:
                    name = ev.key.split("(")[0].split("<")[0].replace("void ", "").replace("thb::", "")
                    per[name] = per.get(name, 0.0) + ev.self_device_time_total / 1e3 / args.reps
            per["total"] = sum(v for k, v in per.items())
            out[key] = per
        return out

    groups = args.groups.split(",") if args.groups else [os.environ.get("THB_CHOL_GROUP", "0")]
    res = {}
    for g in groups:
        os.environ["THB_CHOL_GROUP"] = g
        res[g] = measure()
    name, plim = gpu_description()
    line = dict(gpu=name, power_limit=plim, batch=B, chunk=nb, reps=args.reps, fronts=[dict(np=int(L[q, 5]), w=int(L[q, 10]), b=int(L[q, 11]))
                                                                                       for q in dense],
                direct=os.environ.get("THB_FRONT_BIG_DIRECT", "1") != "0", ms_per_chunk_by_group=res)
    print(json.dumps(line))
    if args.json:
        with open(args.json, "w") as f:
            f.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()
