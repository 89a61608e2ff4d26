#!/usr/bin/env python
"""Summarise an .ncu-rep into a small text file: key raw metrics per kernel
instance plus the top stall instructions of the first instance (needs -lineinfo builds).

    python tools/ncu_summary.py prof.ncu-rep ncu_kv_copy.txt
"""
import csv
import io
import subprocess
import sys

METRICS = [
    "gpu__time_duration.sum", "launch__grid_size", "launch__block_size",
    "launch__registers_per_thread", "launch__occupancy_limit_registers",
    "sm__warps_active.avg.pct_of_peak_sustained_active",
    "dram__bytes_read.sum", "dram__bytes_write.sum",
    "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed",
    "lts__t_bytes.sum", "l1tex__t_bytes.sum",
    "sm__throughput.avg.pct_of_peak_sustained_elapsed",
    "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active",
    "smsp__cycles_active.avg", "sm__cycles_elapsed.max",
    # NVLink: user payload vs protocol overhead, per direction (32-byte granularity)
    "nvltx__bytes.sum", "nvltx__bytes_data_user.sum", "nvltx__bytes_data_protocol.sum",
    "nvlrx__bytes.sum", "nvlrx__bytes_data_user.sum", "nvlrx__bytes_data_protocol.sum",
    "nvltx__bytes_packet_request_data_user.sum", "nvltx__bytes_packet_response_data_user.sum",
    "nvlrx__bytes_packet_request_data_user.sum", "nvlrx__bytes_packet_response_data_user.sum",
]


def run(args):
    return subprocess.run(["ncu", "-i", *args], capture_output=True, text=True).stdout


def main():
    rep, out = sys.argv[1], sys.argv[2]
    lines = [f"# ncu summary of {rep}", ""]
    rows = list(csv.reader(io.StringIO(run([rep, "--page", "raw", "--csv"]))))
    if len(rows) > 2:
        hdr, units = rows[0], rows[1]
        for r in rows[2:]:
            name = r[hdr.index("Kernel Name")]
            lines.append(f"kernel: {name[:140]}")
            vals = {}
            for m in METRICS:
                if m in hdr:
                    i = hdr.index(m)
                    lines.append(f"  {m:62s} {r[i]:>14s} {units[i]}")
                    vals[m] = (r[i], units[i])

            def num(m):
                if m not in vals:
                    return None
                try:
                    v = float(vals[m][0].replace(",", ""))
                except ValueError:
                    return None
                u = vals[m][1].lower()
                scale = {"kbyte": 1e3, "mbyte": 1e6, "gbyte": 1e9, "byte": 1.0,
                         "ns": 1e-9, "us": 1e-6, "usecond": 1e-6, "msecond": 1e-3,
                         "nsecond": 1e-9, "ms": 1e-3, "second": 1.0}.get(u, 1.0)
                return v * scale

            t = num("gpu__time_duration.sum")
            for d in ("tx", "rx"):
                tot, usr = num(f"nvl{d}__bytes.sum"), num(f"nvl{d}__bytes_data_user.sum")
                if t and tot and usr and tot > 0:
                    lines.append(f"  -> NVLink {d}: {tot / t / 1e9:8.1f} GB/s on the wire, "
                                 f"{usr / t / 1e9:8.1f} GB/s user payload, "
                                 f"payload share {100 * usr / tot:5.1f} %")
            lines.append("")
    src = list(csv.reader(io.StringIO(run([rep, "--page", "source", "--csv"]))))
    body, seen = [], 0
    for r in src:
        if r and r[0] == "Kernel Name":
            seen += 1
            if seen > 1:
                break
            continue
        if len(r) > 4 and r[4].isdigit():
            body.append(r)
    total = sum(int(r[4]) for r in body) or 1
    lines.append(f"top stall samples (first instance, {total} samples):")
    for r in sorted(body, key=lambda r: -int(r[4]))[:16]:
        lines.append(f"  {int(r[4]):6d} {100 * int(r[4]) / total:5.1f}%  {r[1].strip()[:100]}")
    mnem = {}
    for r in body:
        op = r[1].strip().split()
        if not op:
            continue
        m = op[1] if op[0].startswith("@") and len(op) > 1 else op[0]
        mnem[m.split(".")[0]] = mnem.get(m.split(".")[0], 0) + 1
    keys = ["LDG", "STG", "UBLKCP", "SYNCS", "MEMBAR", "ERRBAR", "ATOMG", "ATOM", "RED", "BAR", "LDC", "F2FP"]
    lines.append("")
    lines.append("SASS mnemonics present: " + ", ".join(f"{k}x{mnem[k]}" for k in keys if k in mnem))
    open(out, "w").write("\n".join(lines) + "\n")
    print("\n".join(lines[:60]))


if __name__ == "__main__":
    main()
