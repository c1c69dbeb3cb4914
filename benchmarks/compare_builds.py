"""Before/after timing of two source trees on the same GPU: this tree (head) against a plain export of another
(base), usually the parent commit.

Each tree first builds its own library in place (``__graft_entry__.build()``).  Then ``python bench.py ARGS``
runs as a subprocess alternately in the base tree and in this one, ``--rounds`` times each, so drift of a shared
machine hits both sides alike.  Every run passes ``--dump-outputs`` to a temporary directory, and the dumps of all
runs are compared bit for bit with the first base run's.  Prints one JSON line: per side the ``value`` (evals/s)
and ``ms_per_step`` of every round with median / min / max, the same for ``e2e.value`` (the end-to-end rate, which
includes the host's packing and unpacking), the median head / base ratios, each run's clocks
block, whether the outputs are bitwise equal, and the card's name and power limit read in the same call.

    python benchmarks/compare_builds.py --base /path/to/parent-export [--rounds 5] [-- bench.py arguments]

Anything after ``--`` (or any argument this script does not know) is passed to ``bench.py`` unchanged.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile

HEAD = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def card_info() -> dict:
    """Name and power limit of device 0 (read-only query)."""
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=60)
        name, limit = [s.strip() for s in out.stdout.strip().splitlines()[0].split(",")]
        return {"device": name, "power_limit_w": float(limit)}
    except Exception as ex:  # reported, never guessed
        return {"device": None, "power_limit_w": None, "error": f"{type(ex).__name__}: {ex}"}


def build(tree: str) -> None:
    res = subprocess.run([sys.executable, "-c", "import __graft_entry__ as g; g.build()"], cwd=tree,
                         capture_output=True, text=True)
    if res.returncode != 0:
        sys.stderr.write(res.stdout + res.stderr)
        raise SystemExit(f"build failed in {tree}")


def run_bench(tree: str, bench_args: list, dump_dir: str) -> dict:
    cmd = [sys.executable, "bench.py", *bench_args, "--dump-outputs", dump_dir]
    res = subprocess.run(cmd, cwd=tree, capture_output=True, text=True)
    lines = [ln for ln in res.stdout.splitlines() if ln.startswith("{")]
    if res.returncode != 0 or not lines:
        sys.stderr.write(res.stdout[-4000:] + res.stderr[-4000:])
        raise SystemExit(f"bench.py failed in {tree} (exit {res.returncode})")
    return json.loads(lines[-1])


def dumps_equal(a: str, b: str) -> bool:
    import numpy as np

    names = sorted(os.listdir(a))
    if names != sorted(os.listdir(b)) or not names:
        return False
    for n in names:
        x, y = np.load(os.path.join(a, n)), np.load(os.path.join(b, n))
        if x.shape != y.shape or x.tobytes() != y.tobytes():
            return False
    return True


def summary(lines: list) -> dict:
    vals = [ln["value"] for ln in lines]
    e2e = [ln["e2e"]["value"] for ln in lines]
    ms = [ln["ms_per_step"] for ln in lines]
    return {
        "value": vals, "value_median": statistics.median(vals), "value_min": min(vals), "value_max": max(vals),
        "e2e_value": e2e, "e2e_median": statistics.median(e2e), "e2e_min": min(e2e), "e2e_max": max(e2e),
        "ms_per_step": ms, "ms_median": statistics.median(ms), "ms_min": min(ms), "ms_max": max(ms),
        "verified": all(ln.get("verified") for ln in lines),
        "clocks": [ln.get("clocks") for ln in lines],
    }


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0], allow_abbrev=False)
    ap.add_argument("--base", required=True, help="the other source tree (a plain export, not this one)")
    ap.add_argument("--rounds", type=int, default=5, help="bench.py runs per side, alternating")
    ap.add_argument("--no-build", action="store_true", help="use the libraries the trees already hold")
    args, bench_args = ap.parse_known_args()
    bench_args = [a for a in bench_args if a != "--"]
    base = os.path.abspath(args.base)
    if os.path.realpath(base) == os.path.realpath(HEAD):
        raise SystemExit("--base must be another tree than this one")
    if not os.path.exists(os.path.join(base, "bench.py")):
        raise SystemExit(f"{base} has no bench.py")

    card = card_info()
    if not args.no_build:
        build(base)
        build(HEAD)
    runs = {"base": [], "head": []}
    equal = True
    with tempfile.TemporaryDirectory(prefix="compare_builds_") as tmp:
        first = None
        for r in range(args.rounds):
            for side, tree in (("base", base), ("head", HEAD)):
                d = os.path.join(tmp, f"{side}{r}")
                runs[side].append(run_bench(tree, bench_args, d))
                if first is None:
                    first = d
                else:
                    equal = equal and dumps_equal(first, d)
                print(f"[compare_builds] round {r} {side}: {runs[side][-1]['value']:.3f} evals/s", file=sys.stderr, flush=True)
    b, h = summary(runs["base"]), summary(runs["head"])
    line = {
        "bench_args": bench_args,
        "rounds": args.rounds,
        "base": b,
        "head": h,
        "ratio_head_over_base": h["value_median"] / b["value_median"],
        "e2e_ratio_head_over_base": h["e2e_median"] / b["e2e_median"],
        "every_head_faster": min(h["value"]) > max(b["value"]),
        "outputs_bitwise_equal": equal,
        "card": card,
    }
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
