"""Turns the round-end GPU pass (tools/final_gpu_run.sh -> gpurun_out/<R>_*) into the committed profiles/ files.
usage: python tools/make_profiles.py r02"""
import collections
import csv
import json
import os
import shutil
import subprocess
import sys

R = sys.argv[1] if len(sys.argv) > 1 else "r02"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
G, P = os.path.join(ROOT, "gpurun_out"), os.path.join(ROOT, "profiles")

for f in ("bench.json", "bench_reference.json", "bench_g1.json", "bench_three_humanoids.json", "bench_convex_mesh.json", "bench_2gpu.json", "gpu_tests.log", "launches.csv"):
  src = os.path.join(G, f"{R}_{f}")
  if os.path.exists(src):
    shutil.copyfile(src, os.path.join(P, f"{R}_{f}"))

# ---- launch list of the bench command
rows = [r for r in csv.reader(open(os.path.join(G, f"{R}_launches.csv"))) if len(r) > 14 and r[0].isdigit()]
agg = collections.OrderedDict()
for r in rows:
  a = agg.setdefault(r[4], [0, 0.0])
  a[0] += 1
  a[1] += float(r[14]) / 1e3
tot = sum(a[1] for a in agg.values())
with open(os.path.join(P, f"{R}_launches.md"), "w") as f:
  f.write(f"# ncu launch list of `bench.py --no-graph --steps 8 --warmup 3 --no-cpu` (gpu__time_duration.sum, --clock-control none; cold-cache, serialised)\n\n")
  f.write("The step is pipelined over two halves of the 8192 worlds, so every step kernel appears twice per step.\n\n| kernel | launches | mean us | share |\n|---|---|---|---|\n")
  for k, (n, t) in sorted(agg.items(), key=lambda kv: -kv[1][1]):
    f.write(f"| {k[:90]} | {n} | {t / n:.1f} | {t / tot:.3f} |\n")

# ---- per-kernel ncu --set full summary + source hot spots
raw = list(csv.reader(open(os.path.join(G, f"{R}_raw.csv"))))
hdr, idx = raw[0], {h: i for i, h in enumerate(raw[0])}
cols = ["gpu__time_duration.sum", "smsp__inst_executed.sum", "smsp__thread_inst_executed_per_inst_executed.ratio", "dram__bytes_read.sum", "dram__bytes_write.sum",
        "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "sm__warps_active.avg.pct_of_peak_sustained_active", "smsp__issue_active.avg.pct_of_peak_sustained_active",
        "smsp__average_warp_latency_per_inst_issued.ratio", "launch__registers_per_thread", "launch__shared_mem_per_block_dynamic", "launch__block_size", "launch__grid_size",
        "launch__occupancy_limit_shared_mem", "launch__occupancy_limit_registers", "launch__waves_per_multiprocessor", "l1tex__t_sector_hit_rate.pct"]
st = [h for h in hdr if "smsp__average_warps_issue_stalled" in h and h.endswith("per_issue_active.ratio")]
traffic, winst = {}, {}
with open(os.path.join(P, f"{R}_kernels.md"), "w") as f:
  f.write(f"# ncu --set full --clock-control none, {R} kernels (humanoid, 8192 worlds, one GPU, MJB_SPLIT=1 so each kernel covers all worlds; step 120 from the squat keyframe, the middle of the bench window)\n\n")
  f.write("Units as ncu reports them (time us, DRAM Mbyte, shared memory Kbyte/block).  `thread_inst / inst` = average active lanes per warp instruction.\n\n")
  f.write("| kernel | " + " | ".join(c.split("__")[-1].replace(".sum", "").replace(".avg.pct_of_peak_sustained_", " % ").replace(".ratio", "")[:34] for c in cols) + " | top stalls (warps per issue-active cycle) |\n")
  f.write("|---|" + "---|" * (len(cols) + 1) + "\n")
  for r in raw[2:]:
    name = r[idx["Kernel Name"]].replace("void <unnamed>::", "").replace("<unnamed>::", "").split("(")[0]
    vals = sorted([(float(r[idx[h]]), h.split("stalled_")[1].split("_per")[0]) for h in st], reverse=True)[:4]
    f.write(f"| {name} | " + " | ".join(f"{float(r[idx[c]]):.4g}" if c in idx and r[idx[c]] else "" for c in cols) + " | " + ", ".join(f"{n} {v:.2f}" for v, n in vals) + " |\n")
    key = "k_" + name.split("<")[0].replace("k_", "").replace("euler_flat", "euler")
    traffic[key] = (float(r[idx["dram__bytes_read.sum"]]) + float(r[idx["dram__bytes_write.sum"]])) * 1e6
    winst[key] = float(r[idx["smsp__inst_executed.sum"]])
  f.write("\n")
  out = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "ncu_summary.py"), os.path.join(G, f"{R}_raw.csv"), os.path.join(G, f"{R}_src.csv"), "14"], capture_output=True, text=True).stdout
  sect = [l for l in out.splitlines() if not l.startswith("   ") and not l.startswith("== ")]
  f.write("## top source lines by stall samples (per kernel and source file: % of the file's instructions, % of its stall samples, stall classes)\n\n```\n" + "\n".join(l[:200] for l in sect) + "\n```\n")
json.dump({"source": f"ncu --set full, profiles/{R}_kernels.md (dram__bytes_read.sum + dram__bytes_write.sum per launch, bytes; smsp__inst_executed.sum per launch; 8192 worlds)", "traffic_bytes": traffic, "warp_inst": winst},
          open(os.path.join(P, f"{R}_traffic.json"), "w"), indent=1)

# ---- SASS evidence of the bulk-async (TMA) staging
so = os.path.join(ROOT, "mujoco_warp_b200", "libmjb200.so")
sass = subprocess.run(["cuobjdump", "-sass", so], capture_output=True, text=True).stdout
fn, counts = None, collections.OrderedDict()
for line in sass.splitlines():
  if "Function :" in line:
    fn = line.split("Function :")[1].strip()
  for mn in ("UBLKCP", "SYNCS.ARRIVE.TRANS64", "SYNCS.PHASECHK", "FENCE.VIEW.ASYNC", "UTMALDG", "LDGSTS"):
    if fn and mn in line:
      counts.setdefault(fn, collections.Counter())[mn] += 1
with open(os.path.join(P, f"{R}_sass_tma.md"), "w") as f:
  f.write("# Bulk-async (1-D TMA) staging in the shipped SASS (`cuobjdump -sass mujoco_warp_b200/libmjb200.so`)\n\n")
  f.write("`cp.async.bulk` appears as `UBLKCP` (global -> shared with `.S.G`, shared -> global with `.G.S`), the mbarrier transaction count as `SYNCS.ARRIVE.TRANS64`, the wait as\n`SYNCS.PHASECHK.TRANS64.TRYWAIT`, the generic -> async proxy fence as `FENCE.VIEW.ASYNC`.  Instruction counts per kernel:\n\n| kernel | UBLKCP | SYNCS.ARRIVE.TRANS64 | SYNCS.PHASECHK | FENCE.VIEW.ASYNC |\n|---|---|---|---|---|\n")
  for k, c in counts.items():
    if c["UBLKCP"]:
      f.write(f"| `{k[:110]}` | {c['UBLKCP']} | {c['SYNCS.ARRIVE.TRANS64']} | {c['SYNCS.PHASECHK']} | {c['FENCE.VIEW.ASYNC']} |\n")
  ex = [l for l in sass.splitlines() if "UBLKCP" in l][:6]
  f.write("\nexcerpt:\n```\n" + "\n".join(l.rstrip()[:150] for l in ex) + "\n```\n")
print("profiles written:", sorted(x for x in os.listdir(P) if x.startswith(R)))

# ---- where the solver's warp instructions go: per source line of the `--page source` export, grouped by function through marker comments
# found in k_solver.cu itself (`// force/state per row`, `template <int N, bool ELL>` ...), so the table follows the file as it changes
def solver_lines():
  src = os.path.join(G, f"{R}_src.csv")
  rows, cur, fn, hdr, data = list(csv.reader(open(src))), None, None, None, []
  for r in rows:
    if len(r) >= 2 and r[0] == "File Path":
      cur = r[1].split("/")[-1]
    elif len(r) >= 2 and r[0] == "Function Name":
      fn = r[1]
    elif len(r) > 8 and r[0] == "Line No":
      hdr = r
      ii, wi = hdr.index("Instructions Executed"), hdr.index("Warp Stall Sampling (All Samples)")
    elif hdr is not None and len(r) > ii and r[0].isdigit() and fn and "k_solver" in fn:
      try:
        data.append((cur, int(r[0]), r[1].strip()[:110], int(r[ii] or 0), int(r[wi] or 0)))
      except ValueError:
        pass
  agg = collections.OrderedDict()
  for f_, l, s_, i, w in data:
    a = agg.setdefault((f_, l), [s_, 0, 0])
    a[1] += i
    a[2] += w
  ti, ts = sum(v[1] for v in agg.values()) or 1, sum(v[2] for v in agg.values()) or 1
  text = open(os.path.join(ROOT, "mujoco_warp_b200", "csrc", "k_solver.cu")).read().split("\n")
  marks = [("set-up: layout, reductions, row evaluation helpers", 1)]
  for name, needle in (("mul_m", "// res = M vec"), ("update_constraint (force / state per row, J^T force)", "// force/state per row"), ("update_grad", "// grad = Ma"),
                       ("Hessian update in registers (newton_direction_reg)", "// Newton direction for nv <= 32"), ("update_search (dispatch, nv > 32 path)", "// H += sum_list"),
                       ("line search", "template <bool ELL, int NW>\n__device__ __forceinline__ P3 eval_total"), ("CG direction", "// Conjugate-gradient direction"),
                       ("kernel: staging, init_context, main loop, results", "template <bool ELL, bool BIG, bool CG, int NW>\n__global__")):
    pos = "\n".join(text).find(needle)
    if pos >= 0:
      marks.append((name, "\n".join(text)[:pos].count("\n") + 1))
  marks.sort(key=lambda x: x[1])
  grp = collections.OrderedDict((n, 0) for n, _ in marks)
  byfile = collections.Counter()
  for (f_, l), v in agg.items():
    byfile[f_] += v[1]
    if f_ == "k_solver.cu":
      name = [n for n, a in marks if a <= l][-1]
      grp[name] += v[1]
  nworld = 8192
  with open(os.path.join(P, f"{R}_solver_lines.md"), "w") as f:
    f.write(f"# k_solver: warp instructions per world by source ({R}, ncu source counters of the same capture as {R}_kernels.md; humanoid, 8192 worlds)\n\n")
    f.write(f"total {ti / nworld:.0f} warp instructions per world.\n\n| source file | per world | share |\n|---|---|---|\n")
    for k, v in byfile.most_common():
      f.write(f"| {k} | {v / nworld:.0f} | {v / ti:.3f} |\n")
    f.write("\n`mjb_chol.cuh` = Cholesky sweep + substitutions; `mjb_math.cuh` / `sm_30_intrinsics.hpp` = warp reductions and shuffles.\n\n| part of k_solver.cu | per world | share of the kernel |\n|---|---|---|\n")
    for k, v in grp.items():
      f.write(f"| {k} | {v / nworld:.0f} | {v / ti:.3f} |\n")
    f.write("\n## top lines by instructions\n\n```\n")
    for (f_, l), v in sorted(agg.items(), key=lambda x: -x[1][1])[:40]:
      f.write(f"{v[1] / nworld:7.1f} inst/world {v[1] / ti * 100:5.1f}%i {v[2] / ts * 100:5.1f}%stall  {f_}:{l:<4d} {v[0]}\n")
    f.write("```\n")


try:
  solver_lines()
except Exception as e:  # the source page is optional
  print("solver_lines skipped:", e)
