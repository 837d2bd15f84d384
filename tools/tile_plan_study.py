"""Planner check of the tiled sweep kernel: on each shipped geometry, time every feasible chunk count (sweep_chunks, the
B200_SWEEP_CHUNKS knob) x y-tile layout (B200_TILE_TAIL) on the bench's loop-closure batch, and set the planner's own pick
against the fastest plan measured.

A setting is timed as `--repeats` uploads, each timed over `--runs` launches after one warm-up (minimum kernel time per upload);
the spread of a plan is (max - min) / median over its repeats.  Settings that plan the same (chunks, bands, layout) are timed once.

usage: tile_plan_study.py [--n 1000] [--geoms 4:12,8:12,4:20,8:20] [--repeats 3] [--runs 5] [--json OUT]
"""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1000, help="candidate scans (pairs)")
    ap.add_argument("--geoms", default="4:12,8:12,4:20,8:20", help="search dimension [m]:range threshold [m], comma separated")
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--max-chunks", type=int, default=21)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()

    import bench
    from slam_toolbox_b200 import api
    qr, qp, cr, cp, cs = bench.make_inputs(0, a.n, 1, 1)
    laser = api.LaserRangeFinder()
    mapper = api.MapperParams(**{k: (bool(v) if k == "use_response_expansion" else v) for k, v in bench.LOOP_MAPPER.items()})
    dev = bench.device_info(0)

    def timed(dim, rt, chunks, tail, seen):
        """(plan key, plan, timings) of one setting; no timings when its plan is one of `seen`"""
        os.environ["B200_TILE_TAIL"] = str(tail)
        sm = api.ScanMatcher.Create(mapper, dim, 0.05, 0.03, rt)
        sm.set_option("sweep_kernel", 2)
        sm.set_option("sweep_chunks", chunks)
        per = []
        plan = key = None
        for _ in range(a.repeats):
            sm.batch_upload(api.ScanBlock(qr, qp, laser), api.ScanBlock(cr, cp, laser), cs, None, False)
            info, plan = sm.batch_info(), sm.batch_tile_info()
            assert info["kernel"] == "tile", info
            key = (plan["chunks"], plan["bands"], plan["tail"], plan["cluster"])
            if key in seen:
                sm.close()
                return key, plan, None
            sm.batch_run()
            ms = []
            for _ in range(a.runs):
                sm.batch_run()
                ms.append(sm.batch_kernel_ms())
            per.append(min(ms))
        sm.close()
        med = statistics.median(per)
        return key, plan, {"ms": [round(x, 4) for x in per], "median_ms": round(med, 4),
                           "spread_pct": round(100.0 * (max(per) - min(per)) / med, 3)}

    out = {"gpu": dev.get("name"), "power_limit_w": dev.get("power_limit_w"), "max_sm_clock_mhz": dev.get("sm_max_mhz"),
           "pairs": a.n, "repeats": a.repeats, "runs": a.runs, "geometries": []}
    for g in a.geoms.split(","):
        dim, rt = (float(v) for v in g.split(":"))
        seen, plans = set(), []
        key, plan, t = timed(dim, rt, 0, 1, seen)
        pick = {"plan": plan, **t}
        seen.add(key)
        plans.append({"setting": "auto", "plan": plan, **t})
        for tail in (1, 0):
            for chunks in range(1, a.max_chunks + 1):
                key, plan, t = timed(dim, rt, chunks, tail, seen)
                if t is None:
                    continue
                seen.add(key)
                plans.append({"setting": f"chunks>={chunks} tail={tail}", "plan": plan, **t})
        best = min(plans, key=lambda p: p["median_ms"])
        within = pick["median_ms"] - best["median_ms"] <= best["median_ms"] * max(best["spread_pct"], pick["spread_pct"]) / 100.0
        row = {"geom": g, "pick": pick, "best": best, "pick_over_best": round(pick["median_ms"] / best["median_ms"], 4),
               "pick_within_spread": bool(within), "plans": plans}
        out["geometries"].append(row)
        print(f"{g}: pick {pick['plan']['chunks']} chunks / {pick['plan']['bands']} bands / tail {pick['plan']['tail']} "
              f"{pick['median_ms']:.3f} ms (+-{pick['spread_pct']:.2f} %); best {best['setting']} {best['plan']['chunks']} chunks / "
              f"{best['plan']['bands']} bands {best['median_ms']:.3f} ms (+-{best['spread_pct']:.2f} %); within spread: {within}",
              flush=True)
    print(json.dumps(out))
    if a.json:
        with open(a.json, "w") as fh:
            json.dump(out, fh, indent=1)


if __name__ == "__main__":
    main()
