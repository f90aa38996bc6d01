"""Reads `ncu -i <rep> --page raw --csv` (stdin or file) of tools/ncu_targets.py and writes
  profiles/<prefix>_ncu_top_kernels_summary.txt   one line per captured kernel: duration, DRAM read/write bytes, tensor-pipe activity,
                                                  DRAM throughput %, registers
  profiles/<prefix>_ncu_gemm_traffic.json         {"signatures": {"M,N,K,a_mn,b_mn,act,res,atomic": dram bytes per launch}}
                                                  (GEMM launches are attributed in launch order with profiles/ncu_targets_order.json)
No GPU needed:  ncu -i x.ncu-rep --page raw --csv | python tools/ncu_summary.py <prefix>"""
import csv, json, os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
prefix = sys.argv[1]
rows = list(csv.reader(sys.stdin))
hdr = None
for i, r in enumerate(rows):
    if "Kernel Name" in r:
        hdr, body = r, rows[i + 2:]      # the line after the header holds the units
        units = rows[i + 1]
        break
assert hdr, "no ncu raw csv header found"
col = {n: i for i, n in enumerate(hdr)}
def f(r, name):
    try:
        return float(r[col[name]].replace(",", ""))
    except Exception:
        return None
def to_bytes(r, name):
    v = f(r, name)
    u = units[col[name]].lower() if name in col else ""
    if v is None: return None
    return v * {"byte": 1, "kbyte": 1e3, "mbyte": 1e6, "gbyte": 1e9}.get(u, 1)
order = json.load(open(os.path.join(ROOT, "profiles", "ncu_targets_order.json")))
out, sigs, gi = [], {}, 0
for r in body:
    if len(r) < len(hdr): continue
    name = r[col["Kernel Name"]]
    dur = f(r, "gpu__time_duration.sum")
    du = units[col["gpu__time_duration.sum"]]
    dur_us = dur * {"ns": 1e-3, "us": 1, "ms": 1e3, "nsecond": 1e-3, "usecond": 1, "msecond": 1e3}.get(du, 1e-3)
    rd, wr = to_bytes(r, "dram__bytes_read.sum"), to_bytes(r, "dram__bytes_write.sum")
    tens = f(r, "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active") if "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active" in col else None
    dthr = f(r, "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed") if "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed" in col else None
    regs = f(r, "launch__registers_per_thread")
    tag = ""
    if "gemm_wgmma" in name and gi < len(order):
        tag = order[gi]["tag"]
        sigs[",".join(str(x) for x in order[gi]["sig"])] = (rd or 0) + (wr or 0)
        gi += 1
    short = name.split("(")[0][-70:]
    out.append(f"{short:72s} {dur_us:8.1f} us  dram rd {rd / 1e6 if rd is not None else -1:8.2f} MB wr {wr / 1e6 if wr is not None else -1:8.2f} MB  "
               f"tensor pipe {tens if tens is not None else -1:5.1f} %  dram thr {dthr if dthr is not None else -1:5.1f} %  regs {regs}  {tag}")
open(os.path.join(ROOT, "profiles", prefix + "_ncu_top_kernels_summary.txt"), "w").write("\n".join(out) + "\n")
json.dump(dict(source=prefix + " ncu --set full capture of tools/ncu_targets.py (cold cache, one launch each)", signatures=sigs),
          open(os.path.join(ROOT, "profiles", prefix + "_ncu_gemm_traffic.json"), "w"), indent=1)
print("\n".join(out))
