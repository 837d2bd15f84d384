"""Wavefront and instruction account of k_sweep_tile's correlation loops: a lower bound in SM cycles per pair.

Two inputs, multiplied together:
  * the per-trip cost of every correlation loop, read from the SASS of the built library (cuobjdump -xelf + nvdisasm -g): the
    innermost loops (back-edge branches) are matched to the loops of sm_tile.cu by their source lines, an unrolled loop is
    divided by its unroll factor (its shared loads over the loads of one trip);
  * the trips of each loop per pair, counted on the GPU by a build with -DB200_TILE_COUNTS (lane 0 of every warp counts the
    items, the flushes that reduce something and the trips of each loop).  The trips depend only on the plan and the descriptor
    lists, so one count serves every build of the same plan.

Each trip is charged to three resources of an SM (4 sub-partitions):
  * LSU: shared-memory wavefronts, 1 per SM cycle.  Every LDS of the loops is one wavefront: the data loads are conflict-free
    warp-wide LDS.32 (8 rows x 4 words on 32 banks), the descriptor loads broadcast;
  * issue: one warp instruction per sub-partition cycle, 4 per SM cycle;
  * the integer ALU pipe (IADD3, LOP3, PRMT, SHF, LEA, ISETP, SEL, MOV, ...): 16 lanes per sub-partition, 2 warp instructions per
    SM cycle.  IMAD runs on the FMA pipe (same rate), reported beside it.
The bound is the largest of these, summed over the loops; tools/tile_timers.py measures the section ("items: correlation") it
bounds.  The rest of that section (queue pop, item decode, loop set-up) is not in the bound.

usage:
  tile_loop_account.py --sass [--lib LIB]                  per-trip SASS counts of the shipped instantiations (no GPU)
  tile_loop_account.py --count --geom 4:12 [--json OUT]    count the trips per pair on the GPU, then account
  tile_loop_account.py --counts JSON [--lib LIB] [--timers TIMERS_JSON] [--json OUT]
                                                           account a committed count against a library (no GPU)
"""
import argparse
import ctypes as C
import glob
import json
import os
import re
import subprocess
import sys
import tempfile
from collections import Counter
from concurrent.futures import ThreadPoolExecutor

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from slam_toolbox_b200 import build as _build  # noqa: E402

SRC = os.path.join(_build.CSRC, "sm_tile.cu")
K_MAIN = 5   # row tiles of the main part of a y-tile on the tail layout (both shipped geometries run it)

# counters of the -DB200_TILE_COUNTS build, in the order of the kernel's kCn* enum
COUNTERS = ["item", "flush", "plain4", "plain2", "plain1", "single", "pair", "tail_plain", "tail_single", "tail_pair", "edge"]

# correlation loops: source header, shared loads of one trip (data + descriptor) on the tail layout
LOOPS = {
    "plain4": (r"for \(; b \+ 3 < pe; b \+= 4\)", 4 * K_MAIN + 1),
    "plain2": (r"for \(; b \+ 1 < pe; b \+= 2\)", 2 * K_MAIN + 1),
    "single": (r"for \(int k = pe; k < se; k \+= 2\)", K_MAIN + 1),
    "pair": (r"for \(int k = ps; k < pe2; k \+= 4\)", 2 * K_MAIN + 1),
    "tail_plain": (r"for \(int k = b\w* \+ y_l; k < pe; k \+= 8\)", 2),
    "tail_single": (r"for \(int k = pe \+ 2 \* y_l; k < se; k \+= 16\)", 2),
    "tail_pair": (r"for \(int k = ps \+ 4 \* y_l; k < pe2; k \+= 32\)", 3),
    "edge": (r"for \(int k = 0; k < cn; \+\+k\)", K_MAIN + 1),
}
# the odd plain beam is straight-line code, not a loop: charged with its loads and the ALU work of one row-tile step per row tile
STRAIGHT = {"plain1": (r"if \(b < pe\) \{", K_MAIN + 1)}

ALU = {"IADD3", "LOP3", "PRMT", "SHF", "LEA", "ISETP", "SEL", "IMNMX", "VIMNMX", "MOV", "P2R", "R2P", "PLOP3", "IABS", "BMSK",
       "SGXT", "FLO", "POPC", "BREV", "CS2R", "S2R", "VIADD"}
FMA = {"IMAD", "IMUL", "IADD", "FFMA", "FADD", "FMUL"}
LDS = {"LDS"}

# the shipped geometries run these instantiations: sub-grid pitch 76 words (4 m / 12 m) and 132 (8 m / 20 m), tail layout
FUNCS = {"4:12": "_ZN4b20012k_sweep_tileILi76ELb1EEEvNS_8SweepDevENS_7TileDevE",
         "8:20": "_ZN4b20012k_sweep_tileILi132ELb1EEEvNS_8SweepDevENS_7TileDevE"}


def _block_end(lines, i):
    """Last line (1-based) of the brace block opened on line i (0-based index)."""
    depth = 0
    for j in range(i, len(lines)):
        depth += lines[j].count("{") - lines[j].count("}")
        if depth <= 0 and j > i:
            return j + 1
    raise ValueError(f"unbalanced block at line {i + 1}")


def source_ranges(src=SRC):
    lines = open(src).read().splitlines()
    k0 = next(i for i, ln in enumerate(lines) if "k_sweep_tile(SweepDev" in ln)
    k1 = next(i for i, ln in enumerate(lines) if i > k0 and ln.startswith("// host side"))
    ranges = {}
    for kind, (pat, _) in list(LOOPS.items()) + list(STRAIGHT.items()):
        hits = [i for i in range(k0, k1) if re.search(pat, lines[i])]
        if kind == "plain1":
            hits = hits[:1]   # the first `if (b < pe) {` of the kernel is the odd plain beam
        if len(hits) != 1:
            raise ValueError(f"{kind}: {len(hits)} matches of its loop header in {src}")
        ranges[kind] = (hits[0] + 1, _block_end(lines, hits[0]))
    ranges["_helpers"] = (1, k0)   # the inlined helpers above the kernel (lds_u32, odd_bytes_t, ...) carry their own lines
    return ranges


def disassemble(lib, func):
    """[(addr, opcode, operands, source line or None, label or None)] of one function, from the library's sm_90a cubin, and the
    path of the sm_tile.cu it was compiled from (its line numbers are that file's)."""
    with tempfile.TemporaryDirectory() as tmp:
        subprocess.run(["cuobjdump", "-xelf", "all", os.path.abspath(lib)], cwd=tmp, check=True, stdout=subprocess.DEVNULL)
        for cub in sorted(glob.glob(os.path.join(tmp, "*.cubin"))):
            out = subprocess.run(["nvdisasm", "-g", "-c", cub], capture_output=True, text=True).stdout
            if f"\n{func}:" in out:
                break
        else:
            raise RuntimeError(f"{func} not found in {lib}")
    body = out.split(f"\n{func}:", 1)[1]
    ins, line, label, src = [], None, None, None
    for ln in body.splitlines()[1:]:
        if ln.strip() == f".text.{func}:":
            continue
        if ln.startswith(".text.") or (ln and not ln[0].isspace() and ln.endswith(":") and not ln.startswith(".L")):
            break   # next section / function
        m = re.match(r'\s*//## File "(.*)", line (\d+)', ln)
        if m:
            line = int(m.group(2)) if m.group(1).endswith("sm_tile.cu") else None
            src = src or (m.group(1) if m.group(1).endswith("sm_tile.cu") else None)
            continue
        m = re.match(r"(\.L_x_\d+):", ln.strip())
        if m:
            label = m.group(1)
            continue
        m = re.match(r"\s*/\*([0-9a-f]+)\*/\s+(@!?U?P\w+\s+)?([A-Z][A-Z0-9_.]*)(.*);", ln)
        if m:
            ins.append((int(m.group(1), 16), m.group(3), m.group(4), line, label))
            label = None
    return ins, src


def _pipe(op):
    base = op.split(".")[0]
    return "lds" if base in LDS else "alu" if base in ALU else "fma" if base in FMA else "other"


def sass_blocks(lib, func):
    """Per-trip SASS counts of every correlation loop of one instantiation."""
    ins, src = disassemble(lib, func)
    ranges = source_ranges(src if src and os.path.exists(src) else SRC)
    addr_of = {lab: a for a, _, _, _, lab in ins if lab}
    loops = []
    for a, op, rest, _, _ in ins:
        if op.startswith("BRA"):
            m = re.search(r"`\((\.L_x_\d+)\)", rest)
            if m and m.group(1) in addr_of and addr_of[m.group(1)] <= a:
                loops.append((addr_of[m.group(1)], a))
    inner = [lp for lp in loops if not any(o != lp and lp[0] <= o[0] and o[1] <= lp[1] for o in loops)]
    res = {}
    for lo, hi in inner:
        body = [x for x in ins if lo <= x[0] <= hi]
        votes = Counter(k for _, _, _, ln, _ in body for k, (r0, r1) in ranges.items() if ln is not None and r0 <= ln <= r1 and k in LOOPS)
        if not votes:
            continue
        kind = votes.most_common(1)[0][0]
        pipes = Counter(_pipe(op) for _, op, _, _, _ in body)
        ops = Counter(op.split(".")[0] for _, op, _, _, _ in body)
        unroll = max(1, round(pipes["lds"] / LOOPS[kind][1]))
        blk = {"instructions": len(body), "lds": pipes["lds"], "alu": pipes["alu"], "fma": pipes["fma"], "other": pipes["other"],
               "prmt": ops["PRMT"], "imad": ops["IMAD"], "iadd3": ops["IADD3"], "unroll": unroll}
        # an unrolled copy and its remainder loop: keep the steady-state (most unrolled) one
        if kind not in res or unroll > res[kind]["unroll"]:
            res[kind] = blk
    # the odd plain beam: the instructions of its source range, and those of the inlined helpers (its loads and byte extracts carry
    # the helpers' lines) between its first and last instruction.  An estimate: the scheduler may interleave neighbouring code
    r0, r1 = ranges["plain1"]
    h0, h1 = ranges["_helpers"]
    own = [a for a, _, _, ln, _ in ins if ln is not None and r0 <= ln <= r1]
    span = [x for x in ins if own and min(own) <= x[0] <= max(own) and x[3] is not None and (r0 <= x[3] <= r1 or h0 <= x[3] <= h1)]
    cnt = Counter(_pipe(op) for _, op, _, _, _ in span)
    ops = Counter(op.split(".")[0] for _, op, _, _, _ in span)
    n_lds = STRAIGHT["plain1"][1]
    res["plain1"] = {"instructions": sum(cnt.values()) + n_lds - cnt["lds"], "lds": n_lds, "alu": cnt["alu"], "fma": cnt["fma"],
                     "other": cnt["other"], "prmt": ops["PRMT"], "imad": ops["IMAD"], "iadd3": ops["IADD3"], "unroll": 1}
    for kind in list(LOOPS):
        if kind not in res:
            raise RuntimeError(f"no SASS loop found for {kind} in {func}")
    per_trip = {}
    for kind, b in res.items():
        u = b["unroll"]
        per_trip[kind] = {k: round(v / u, 3) for k, v in b.items() if k != "unroll"}
        per_trip[kind]["unroll"] = u
    return per_trip


def account(per_trip, trips_per_pair):
    tot = Counter()
    for kind, t in trips_per_pair.items():
        if kind in per_trip:
            for k in ("instructions", "lds", "alu", "fma"):
                tot[k] += t * per_trip[kind][k]
    bound = {"lsu_wavefronts": tot["lds"], "issue": tot["instructions"] / 4.0, "alu_pipe": tot["alu"] / 2.0,
             "fma_pipe": tot["fma"] / 2.0}
    bound = {k: round(v) for k, v in bound.items()}
    bound["binding"] = max(("lsu_wavefronts", "issue", "alu_pipe", "fma_pipe"), key=lambda k: bound[k])
    bound["cycles"] = bound[bound["binding"]]
    return bound


def build_counting(out_dir):
    nvcc = os.environ.get("NVCC", "nvcc")

    def one(unit):
        obj = os.path.join(out_dir, unit.replace(".cu", ".o"))
        subprocess.run([nvcc] + _build.ARCH + _build.COMMON + _build.UNITS[unit] +
                       ["-DB200_TILE_COUNTS", "-c", os.path.join(_build.CSRC, unit), "-o", obj], check=True)
        return obj

    with ThreadPoolExecutor(len(_build.UNITS)) as ex:
        objs = list(ex.map(one, _build.UNITS))
    lib = os.path.join(out_dir, "libb200slam_counts.so")
    subprocess.run([nvcc] + _build.ARCH + ["-shared", "--cudart", "shared", "-Xlinker", "-rpath,/usr/local/cuda/lib64",
                                           "-o", lib] + objs + ["-ldl"], check=True)
    return lib


def count_trips(geom, n, build_dir, reuse):
    """Trips per pair of every loop on the bench's loop-closure batch (1 query x n candidates) at one geometry (GPU)."""
    prebuilt = os.path.join(build_dir, "libb200slam_counts.so")
    _build.LIB = prebuilt if (reuse and os.path.exists(prebuilt)) else build_counting(build_dir)
    import bench
    from slam_toolbox_b200 import api
    L = api.lib()
    L.b200_tile_counts.argtypes = [C.POINTER(C.c_ulonglong), C.c_int]
    L.b200_tile_counts.restype = C.c_int
    nc = L.b200_tile_counts(None, 1)
    assert nc == len(COUNTERS), nc
    dim, rt = (float(v) for v in geom.split(":"))
    qr, qp, cr, cp, cs = bench.make_inputs(0, n, 1, 1)
    laser = api.LaserRangeFinder()
    mapper = api.MapperParams(**{k: (bool(v) if k == "use_response_expansion" else v) for k, v in bench.LOOP_MAPPER.items()})
    sm = api.ScanMatcher.Create(mapper, dim, 0.05, 0.03, rt)
    sm.set_option("sweep_kernel", 2)
    sm.batch_upload(api.ScanBlock(qr, qp, laser), api.ScanBlock(cr, cp, laser), cs, None, False)
    info, plan = sm.batch_info(), sm.batch_tile_info()
    assert info["kernel"] == "tile", info
    L.b200_tile_counts(None, 1)
    sm.batch_run()
    buf = (C.c_ulonglong * nc)()
    assert L.b200_tile_counts(buf, 1) == nc
    sm.close()
    return plan, {k: buf[i] / n for i, k in enumerate(COUNTERS)}


def report(geom, plan, trips, per_trip, timers=None):
    # the loads per trip (LOOPS, K_MAIN) and the instantiations (FUNCS) are those of the tail layout
    if not (plan.get("tail") and plan.get("ytile_rows") == 40):
        raise SystemExit(f"geometry {geom}: the plan runs 48-row y-tiles ({plan}); the account models the tail layout only")
    b = account(per_trip, trips)
    out = {"geom": geom, "plan": plan, "trips_per_pair": {k: round(v, 2) for k, v in trips.items()}, "sass_per_trip": per_trip,
           "bound_cycles_per_pair": b}
    print(f"geometry {geom}: trips per pair and SASS per trip")
    print(f"  {'loop':12s} {'trips':>10s} {'instr':>7s} {'LDS':>5s} {'ALU':>5s} {'IMAD':>5s} {'PRMT':>5s} {'unroll':>6s}")
    for kind, p in per_trip.items():
        print(f"  {kind:12s} {trips.get(kind, 0):10,.0f} {p['instructions']:7.1f} {p['lds']:5.1f} {p['alu']:5.1f} {p['imad']:5.1f} "
              f"{p['prmt']:5.1f} {p['unroll']:6d}")
    print(f"  items {trips['item']:,.0f}, flushes {trips['flush']:,.0f} per pair")
    print(f"  bound (SM cycles per pair): LSU {b['lsu_wavefronts']:,}  issue {b['issue']:,}  ALU {b['alu_pipe']:,}  "
          f"FMA {b['fma_pipe']:,}  -> {b['binding']}")
    if timers:
        t = json.load(open(timers))
        corr = t["split"]["items: correlation"] * t["sm_cycles_per_pair"]
        out["measured_correlation_cycles_per_pair"] = round(corr)
        out["measured_over_bound"] = round(corr / b["cycles"], 3)
        out["timers"] = os.path.basename(timers)
        print(f"  measured correlation {corr:,.0f} cycles per pair ({os.path.basename(timers)}): {corr / b['cycles']:.2f} x the bound")
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sass", action="store_true", help="print the per-trip SASS counts only")
    ap.add_argument("--count", action="store_true", help="count the trips on the GPU")
    ap.add_argument("--counts", default=None, help="a JSON written by --count: take its trips per pair")
    ap.add_argument("--lib", default=_build.LIB, help="library whose SASS is accounted (default: the in-tree build)")
    ap.add_argument("--geom", default="4:12")
    ap.add_argument("--n", type=int, default=1000)
    ap.add_argument("--timers", default=None, help="a tools/tile_timers.py JSON of the same geometry")
    ap.add_argument("--build-dir", default=None)
    ap.add_argument("--reuse", action="store_true")
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    lib = os.path.abspath(a.lib)   # before count_trips points the build module at the counting library
    if a.sass:
        res = {g: sass_blocks(lib, f) for g, f in FUNCS.items()}
        print(json.dumps(res, indent=1))
        return
    if a.count:
        build_dir = a.build_dir or tempfile.mkdtemp(prefix="b200_tile_counts_")
        os.makedirs(build_dir, exist_ok=True)
        plan, trips = count_trips(a.geom, a.n, build_dir, a.reuse)
        geom = a.geom
    else:
        c = json.load(open(a.counts))
        plan, trips, geom = c["plan"], c["trips_per_pair"], c["geom"]
    out = report(geom, plan, trips, sass_blocks(lib, FUNCS[geom]), a.timers)
    out["library"] = os.path.relpath(lib, ROOT) if lib.startswith(ROOT) else os.path.basename(lib)
    if a.json:
        with open(a.json, "w") as fh:
            json.dump(out, fh, indent=1)


if __name__ == "__main__":
    main()
