"""Summarise an Nsight Compute report of tools/profile_update.py into JSON files.

    python tools/ncu_summary.py update.ncu-rep ncu_update.json [traffic.json]

Kernel launches are mapped to the layer they implement by instantiation and order inside one minibatch
(forward conv1-3, fc, heads; backward heads, fc, conv3, conv2, conv1).  The traffic file carries, per layer,
DRAM bytes (dram__bytes_read.sum + dram__bytes_write.sum) next to the algorithmic bytes bench.py reports."""
import csv
import io
import json
import subprocess
import sys

METRICS = ["gpu__time_duration.sum", "dram__bytes_read.sum", "dram__bytes_write.sum",
           "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active",
           "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "sm__throughput.avg.pct_of_peak_sustained_elapsed",
           "lts__t_sector_hit_rate.pct", "launch__registers_per_thread", "launch__grid_size", "launch__block_size",
           "smsp__issue_active.avg.pct_of_peak_sustained_active"]

# algorithmic bytes per sample (DESIGN.md "kernels" table; the same figures as the ProfScope calls in net_tc.cu)
ALGO = {
    "conv1_fwd": (28224 + 12800) * 2 + 1600, "conv2_fwd": (12800 + 5184) * 2 + 648, "conv3_fwd": (5184 + 3136) * 2 + 392,
    "fc_fwd": (3136 + 512) * 2, "fc_dgrad": (3136 + 512) * 2 + 392, "conv3_dgrad": (7744 + 6400 + 7744) * 2 + 648,
    "conv2_dgrad": (7744 + 14112) * 2 + 1600, "conv3_wgrad": (5184 + 5184) * 2, "conv2_wgrad": (12800 + 6400) * 2,
    "conv1_wgrad": (28224 + 14112) * 2, "fc_wgrad": (3136 + 512) * 2,
}
# uint8 rollout (round 2): conv1 reads the frames as bytes (row-major 28224 B forward, channel-major 28672 B for the
# weight gradient whose dY operand is fp16)
ALGO_U8 = {"conv1_fwd": 28224 + 12800 * 2 + 1600, "conv1_wgrad": 28672 + 14112 * 2}


def to_bytes(v, unit):
    return float(v) * {"byte": 1, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9, "Tbyte": 1e12}[unit]


def to_us(v, unit):
    return float(v) * {"ns": 1e-3, "us": 1, "ms": 1e3, "s": 1e6}.get(unit, 1)   # "usecond" style units fall through


def main():
    rep, out = sys.argv[1], sys.argv[2]
    txt = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv", "--metrics", ",".join(METRICS)],
                         capture_output=True, text=True, check=True).stdout
    rows = list(csv.reader(io.StringIO(txt)))
    hdr, units, data = rows[0], rows[1], rows[2:]
    col = {h: i for i, h in enumerate(hdr)}
    seen = {}
    kernels = []
    u8 = any("tc_conv1_i8" in r[col["Kernel Name"]] for r in data)
    algo = dict(ALGO, **ALGO_U8) if u8 else ALGO
    for r in data:
        name = r[col["Kernel Name"]]
        short = name.split("(")[0].replace("void ", "").replace("b200rl::", "").replace("(int)", "")
        grid = int(r[col["launch__grid_size"]])
        k = seen.get(short, 0)
        seen[short] = k + 1
        layer = None
        if short.startswith("tc_conv1_i8"): layer = "conv1_fwd"
        elif short.startswith("tc_conv1_wgrad_u8"): layer = "conv1_wgrad"
        elif short.startswith("tc_conv_win<32"): layer = "conv1_fwd"
        elif short.startswith("tc_conv_win<64, 2"): layer = "conv2_fwd"
        elif short.startswith("tc_conv_win<64, 1"): layer = "conv3_fwd" if k % 2 == 0 else "conv3_dgrad"
        elif short.startswith("tc_conv_win<128"): layer = "conv2_dgrad"
        elif short.startswith("tc_wgrad_win"): layer = ["conv3_wgrad", "conv2_wgrad", "conv1_wgrad"][k % (2 if u8 else 3)]
        elif short.startswith("tc_gemm_tma<256"): layer = "fc_fwd" if k % 2 == 0 else "fc_dgrad"
        elif short.startswith("tc_wgrad_tma"): layer = "fc_wgrad"
        e = {"id": int(r[col["ID"]]), "kernel": short, "layer": layer, "grid": grid,
             "block": int(r[col["launch__block_size"]]), "regs": int(r[col["launch__registers_per_thread"]]),
             "time_us": round(to_us(r[col["gpu__time_duration.sum"]], units[col["gpu__time_duration.sum"]]), 2),
             "dram_read_bytes": int(to_bytes(r[col["dram__bytes_read.sum"]], units[col["dram__bytes_read.sum"]])),
             "dram_write_bytes": int(to_bytes(r[col["dram__bytes_write.sum"]], units[col["dram__bytes_write.sum"]])),
             "tensor_pipe_pct": float(r[col[METRICS[3]]]), "dram_pct_of_peak": float(r[col[METRICS[4]]]),
             "sm_throughput_pct": float(r[col[METRICS[5]]]), "l2_hit_pct": float(r[col[METRICS[6]]]),
             "issue_active_pct": float(r[col[METRICS[10]]])}
        kernels.append(e)
    json.dump({"source": "ncu --set full --clock-control none --profile-from-start off python tools/profile_update.py "
                         "32768 1 [s2d|u8s2d] (one minibatch update at M=32768 + one rollout step at N=1024; under the "
                         "profiler: cold caches, serialised launches)", "kernels": kernels}, open(out, "w"), indent=1)
    if len(sys.argv) > 3:
        n = int(sys.argv[4]) if len(sys.argv) > 4 else 32768
        tr = {"source": f"{out}: dram__bytes_read.sum + dram__bytes_write.sum of the first launch of each layer at "
                        f"minibatch n = {n} (ncu --set full)"}
        for e in kernels:
            if e["layer"] and e["layer"] not in tr and e["time_us"] > 60:      # the n = 32768 launch, not the rollout one
                tr[e["layer"]] = {"n": n, "dram_bytes": e["dram_read_bytes"] + e["dram_write_bytes"],
                                  "algorithmic_bytes": algo[e["layer"]] * n, "kernel": e["kernel"],
                                  "time_us_under_ncu": e["time_us"]}
        json.dump(tr, open(sys.argv[3], "w"), indent=1)
    for e in kernels:
        print(f"{e['id']:3d} {e['kernel'][:34]:34s} {str(e['layer']):12s} {e['time_us']:9.1f} us  dram {1e-9 * (e['dram_read_bytes'] + e['dram_write_bytes']):7.3f} GB  "
              f"tensor {e['tensor_pipe_pct']:5.1f}%  dram {e['dram_pct_of_peak']:5.1f}%  issue {e['issue_active_pct']:5.1f}%")


if __name__ == "__main__":
    main()
