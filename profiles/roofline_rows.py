"""The dominant kernel's true algorithmic bytes for the bucketed detector's row format, from bench.py JSON lines.

bench.py charges 2 B per (fresh subject, receiver) and 4 B per (carried subject, receiver), the size of a uint16 word.  Bucketed
rows hold ring bits only: a byte plane plus a hi plane of 2 bits per receiver at K <= 10 (1.25 B) or 8 bits at K <= 14 (2 B),
padded to whole 1024-receiver tiles (cd_internal.cuh, RowRef).  The sweep kernel keeps uint16 rows (2 B).  This prints, for
`roofline` and `roofline_carried`, the bytes that format moves, the achieved rate over the kernel time bench.py measured and the
fraction of the peak it reports.  It uses only fields of the line: K, receivers, fresh / carried subjects, kernel ms and peak.

    python bench.py ... | python profiles/roofline_rows.py
    python profiles/roofline_rows.py profiles/h100/bench_c5.json
"""
import json
import re
import sys

TILE = 1024
EXTRA_PER_RECEIVER = 5          # flags + blocked byte, read once per receiver (the same term as bench.py)


def row_bytes(K, path):
    """bytes per (subject, receiver) of one row"""
    if path == "sweep":
        return 2.0
    return 1.0 + (2 if K <= 10 else 8) / 8.0


def padded(R, path):
    return R if path == "sweep" else -(-R // TILE) * TILE


def true_bytes(line):
    cfg = line["config"]
    K, R, path = cfg["K"], cfg["receivers_per_gpu"], cfg.get("kernel_path", "bucketed-uniform")
    rb, Rp = row_bytes(K, path), padded(R, path)
    out = {}
    rl = line["roofline"]
    if rl.get("per_batch"):
        fresh = sum(b["fresh_subjects"] for b in rl["per_batch"])
        carried = sum(b["carried_subjects"] for b in rl["per_batch"])
    else:                       # a sequence in one pass: every subject of the stream is written once
        fresh, carried = cfg["subjects"], 0
    launches = rl.get("launches_per_step", 1)
    alg = (rb * fresh + 2 * rb * carried) * Rp + EXTRA_PER_RECEIVER * R * launches
    out["roofline"] = (alg / launches, rl["kernel_ms"], rl["peak"])
    rc = line.get("roofline_carried")
    if rc:
        m = re.search(r"(\d+) carried subjects.*?(\d+) fresh", rc["kernel"])
        sc, sf = int(m.group(1)), int(m.group(2))
        alg2 = (2 * rb * sc + rb * sf) * Rp + EXTRA_PER_RECEIVER * R
        out["roofline_carried"] = (alg2, rc["kernel_ms"], rc["peak"])
    return out


def main(paths):
    streams = [open(p) for p in paths] if paths else [sys.stdin]
    for f in streams:
        for text in f:
            text = text.strip()
            if not text.startswith("{"):
                continue
            line = json.loads(text)
            if "roofline" not in line:
                continue
            print(line["config"]["workload"])
            for name, (alg, ms, peak) in true_bytes(line).items():
                tbs = alg / (ms * 1e-3) / 1e12
                print("  %-16s %7.3f GB per launch  %7.3f ms  %5.2f TB/s  %.2f of %.2f TB/s" % (name, alg / 1e9, ms, tbs, tbs * 1e3 / peak, peak / 1e3))


if __name__ == "__main__":
    main(sys.argv[1:])
