"""Expansion of the K-ring monitoring overlay, measured on the device (MembershipView.overlaySpectrum, DESIGN.md §4.13): the Rapid
paper quotes lambda / 2K < 0.45 for K = 10, lambda the second largest eigenvalue magnitude of the 2K-regular observer graph.

Grid: K in {4, 6, 8, 10, 12, 14} x n in {10^3, 10^4, 10^5, 10^6} over the synthetic endpoints of rapid_b200.workloads; one JSON line
per cell with ratio = lambda / 2K, the residual bound on lambda, the Lanczos steps spent, the device time of the call (CUDA events
around all its steps, the second of two calls: the first loads the module), that time per step, and the bytes one step moves
computed from the shapes (two 4K-byte table rows read and two 8-byte values written per node by the operator, 8 bytes per node and
basis vector read by each of the two re-orthogonalisation passes, averaged over the steps).

    python profiles/overlay_study.py [--max-nodes 1000000] [--scenario] [--out FILE]

--scenario instead follows the ratio configuration by configuration through ClusterSimulation(overlay_quality=True): bench_sim's
crash scenario at 10^4 nodes with 1 % and with 30 % crashed, and its rolling restart (three waves of 1 % leave and rejoin); a
scenario that does not converge says so and lists the configurations it reached.  One more line applies the 30 % cut to the view
directly (applyCut, no consensus), which answers what the overlay of the survivors is whether or not the cluster agrees on that cut.
The rings come from this project's seeded ring hash; its parity with the reference's hash is not pinned (DESIGN §3), and the
spectrum of a seeded-hash ring family does not depend on which good hash it is.  Runs on the GPU only."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

KS = (4, 6, 8, 10, 12, 14)
NS = (1_000, 10_000, 100_000, 1_000_000)


def gpu_card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def step_bytes(n, K, steps):
    """bytes of one Lanczos step from the shapes, averaged over `steps` steps: (operator, re-orthogonalisation)"""
    operator = n * (2 * 4 * K + 8 + 2 * 8)                      # both table rows and t[v] read, v_j and y written
    mean_basis = (steps + 1) / 2.0                              # step j reads j basis vectors, twice
    reorth = n * (2 * 8 * mean_basis + 6 * 8)                   # + y read and written by each pass, v_j and v_{j-1} by the first
    return operator, reorth


def grid(rb, W, card, max_nodes):
    lines = []
    for n in (x for x in NS if x <= max_nodes):
        packed = W.packed_endpoints(0, n)
        for K in KS:
            view = rb.MembershipView.from_packed(K, *packed)
            view.overlaySpectrum()
            sp = view.overlaySpectrum()
            view.close()
            op, re = step_bytes(n, K, sp.steps)
            lines.append({"study": "overlay", "K": K, "nodes": n, "ratio": sp.ratio, "lambda2": sp.lambda2, "lambda_min": sp.lambda_min,
                          "residual": sp.residual, "steps": sp.steps, "device_ms": sp.device_ms, "ms_per_step": sp.device_ms / sp.steps,
                          "random_regular_edge": 2.0 * (2 * K - 1) ** 0.5 / (2 * K),
                          "step_bytes_operator": op, "step_bytes_reorthogonalisation": re,
                          "call_bytes_per_s": (op + re) * sp.steps / (sp.device_ms * 1e-3), "gpu": card,
                          "note": "device_ms: CUDA events around the whole call (all steps, the host's convergence checks between them "
                                  "included); call_bytes_per_s is bytes from shapes over that time, not a kernel's share of peak"})
            print(json.dumps(lines[-1]), flush=True)
    return lines


def scenarios(rb, W, card):
    lines = []
    for name, n, frac in (("crash", 10_000, 0.01), ("crash", 10_000, 0.30), ("rolling", 10_000, 0.01)):
        s = rb.ClusterSimulation(W.packed_endpoints(0, n), W.node_ids(0, n), seed=24, overlay_quality=True)
        gone = W.pick_smallest(n, (3 if name == "rolling" else 1) * int(n * frac), 24)
        if name == "crash":
            for t in gone.tolist():
                s.setFlags(t, 1)
            out = s.run(15)
        else:
            for k in range(3):
                wave = gone[k::3].tolist()
                s.leave(wave)
                s.run(15)
                hi, lo = W.node_ids((1 << 40) + k * len(wave), len(wave))
                for j, t in enumerate(wave):
                    s.rejoin(t, int(hi[j]), int(lo[j]))
                out = s.run(15)
        lines.append({"study": "overlay scenario", "scenario": name, "nodes": n, "fraction": frac, "K": s.K, "gpu": card,
                      "converged": out["converged"],
                      "initial": {"ratio": s.initial_overlay[0], "residual": s.initial_overlay[1]},
                      "configurations": [{"size": h["size"], "cut": len(h["cut"]), "path": h["path"], "ratio": h["overlay_ratio"],
                                          "residual": h["overlay_residual"]} for h in s.history]})
        s.close()
        print(json.dumps(lines[-1]), flush=True)
    n, K = 10_000, 10
    view = rb.MembershipView.from_packed(K, *W.packed_endpoints(0, n))
    before = view.overlaySpectrum()
    view.applyCut(W.pick_smallest(n, int(n * 0.30), 24), want_map=False)
    after = view.overlaySpectrum()
    lines.append({"study": "overlay scenario", "scenario": "applyCut", "nodes": n, "fraction": 0.30, "K": K, "gpu": card,
                  "initial": {"ratio": before.ratio, "residual": before.residual},
                  "configurations": [{"size": view.n, "cut": n - view.n, "ratio": after.ratio, "residual": after.residual}]})
    print(json.dumps(lines[-1]), flush=True)
    return lines


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--max-nodes", type=int, default=NS[-1])
    ap.add_argument("--scenario", action="store_true", help="the ratio through the crash and rolling scenarios instead of the grid")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("overlay_study.py measures on the GPU; no CUDA device is visible")
    import rapid_b200 as rb
    from rapid_b200 import workloads as W
    card = gpu_card()
    lines = scenarios(rb, W, card) if args.scenario else grid(rb, W, card, args.max_nodes)
    if args.out:
        with open(args.out, "w") as f:
            for r in lines:
                f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
