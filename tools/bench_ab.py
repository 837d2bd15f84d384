"""Alternating A/B of bench.py between built trees: every round runs each tree's bench.py once, in the given order, so
that drift of the card (clocks, temperature, neighbours) spreads evenly over the builds.

usage: bench_ab.py --tree parent=DIR --tree change=DIR [--rounds 3] [--json OUT] [-- bench arguments]

Each tree must already be built (``python -c "import __graft_entry__ as g; g.build()"`` inside it).  Prints and writes the
headline and the kernel time of every sweep_rows entry per build: runs, median and spread ((max - min) / median, percent).
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

DEFAULT_BENCH = ["--gpus", "1", "--steps", "20", "--warmup", "3", "--no-graph", "--no-map", "--no-seq", "--no-replay", "--no-cpu"]


def run_bench(tree, bench_args):
    out = subprocess.run([sys.executable, os.path.join(tree, "bench.py")] + bench_args, cwd=tree, capture_output=True, text=True)
    if out.returncode != 0:
        raise RuntimeError(f"bench.py failed in {tree}:\n{out.stdout[-2000:]}\n{out.stderr[-4000:]}")
    return json.loads([ln for ln in out.stdout.splitlines() if ln.startswith("{")][-1])


def stats(xs):
    med = statistics.median(xs)
    return {"runs": [round(x, 4) for x in xs], "median": round(med, 4), "spread_pct": round(100.0 * (max(xs) - min(xs)) / med, 3)}


def main():
    argv = sys.argv[1:]
    bench_args = DEFAULT_BENCH
    if "--" in argv:
        i = argv.index("--")
        argv, bench_args = argv[:i], argv[i + 1:]
    ap = argparse.ArgumentParser()
    ap.add_argument("--tree", action="append", required=True, help="NAME=DIR of a built tree")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--json", default=None)
    a = ap.parse_args(argv)
    trees = [t.split("=", 1) for t in a.tree]
    res = {name: [] for name, _ in trees}
    for rnd in range(a.rounds):
        for name, d in trees:
            line = run_bench(os.path.abspath(d), bench_args)
            res[name].append(line)
            print(f"round {rnd} {name}: {line['value']:.1f} {line['unit']}", flush=True)
    first = res[trees[0][0]][0]
    out = {"gpu": first["device"].get("name"), "power_limit_w": first["device"].get("power_limit_w"),
           "max_sm_clock_mhz": first["device"].get("sm_max_mhz"),
           "command": "bench.py " + " ".join(bench_args) + f"; builds run alternately ({', '.join(n for n, _ in trees)}) x {a.rounds}",
           "clocks": {name: [ln.get("clocks") for ln in lines] for name, lines in res.items()},
           "headline_matches_per_s": {name: stats([ln["value"] for ln in lines]) for name, lines in res.items()}}
    base = trees[0][0]
    for name, _ in trees[1:]:
        out[f"headline_speedup_{name}_vs_{base}"] = round(out["headline_matches_per_s"][name]["median"] /
                                                          out["headline_matches_per_s"][base]["median"], 4)
    rows = []
    for i, row in enumerate(first.get("sweep_rows", [])):
        r = {"workload": row["workload"], "kernel": row.get("kernel"), "plan": row.get("plan")}
        for name, lines in res.items():
            r[f"kernel_ms_{name}"] = stats([ln["sweep_rows"][i]["kernel_ms"] for ln in lines])
            r[f"parity_exact_{name}"] = all(ln["sweep_rows"][i]["parity_exact"] for ln in lines)
        for name, _ in trees[1:]:
            r[f"speedup_{name}_vs_{base}"] = round(r[f"kernel_ms_{base}"]["median"] / r[f"kernel_ms_{name}"]["median"], 4)
        rows.append(r)
    out["sweep_rows"] = rows
    print(json.dumps(out, indent=1))
    if a.json:
        with open(a.json, "w") as fh:
            json.dump(out, fh, indent=1)


if __name__ == "__main__":
    main()
