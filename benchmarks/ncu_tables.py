"""Turn ncu reports into markdown / JSON summaries.

  python benchmarks/ncu_tables.py conv  out/conv_full.ncu-rep   conv.md conv_dram_traffic.json
  python benchmarks/ncu_tables.py list  out/launches.csv        launches.md
  python benchmarks/ncu_tables.py vote  out/vote_full.ncu-rep   vote.md
  python benchmarks/ncu_tables.py top   out/conv_full.ncu-rep   <kernel index> [n]     (hottest source lines)

Captures (see the header each table carries):
  conv: ncu --profile-from-start off --set full --clock-control none --import-source on
        -k regex:"k_conv_tap|k_conv_col" -c 25 -o out/conv_full python benchmarks/profile_step.py 1
  list: ncu --profile-from-start off --metrics gpu__time_duration.sum --clock-control none --csv
        --log-file out/launches.csv python benchmarks/profile_step.py 2
"""
import csv
import json
import subprocess
import sys

LAYERS = ["stem (s2d 4x4)", "layer1.0.conv1", "layer1.0.conv2", "layer1.1.conv1", "layer1.1.conv2",
          "layer2.0.conv1 (s2)", "layer2.0.downsample", "layer2.0.conv2", "layer2.1.conv1", "layer2.1.conv2",
          "layer3.0.conv1", "layer3.0.downsample", "layer3.0.conv2", "layer3.1.conv1", "layer3.1.conv2",
          "layer4.0.conv1", "layer4.0.downsample", "layer4.0.conv2", "layer4.1.conv1", "layer4.1.conv2",
          "fc.0", "conv8s.0", "conv4s.0", "conv2s.0", "convraw.0 (+head)"]
# GMAC per image of each conv launch at 480x640 (real channels, reference graph)
def _gmac():
    def c(h, w, cin, cout, k): return h * w * cin * cout * k * k / 1e9
    g = [c(240, 320, 3, 64, 7)]
    g += [c(120, 160, 64, 64, 3)] * 4
    g += [c(60, 80, 64, 128, 3), c(60, 80, 64, 128, 1), c(60, 80, 128, 128, 3), c(60, 80, 128, 128, 3), c(60, 80, 128, 128, 3)]
    g += [c(60, 80, 128, 256, 3), c(60, 80, 128, 256, 1), c(60, 80, 256, 256, 3), c(60, 80, 256, 256, 3), c(60, 80, 256, 256, 3)]
    g += [c(60, 80, 256, 512, 3), c(60, 80, 256, 512, 1), c(60, 80, 512, 512, 3), c(60, 80, 512, 512, 3), c(60, 80, 512, 512, 3)]
    g += [c(60, 80, 512, 256, 3), c(60, 80, 256 + 128, 128, 3), c(120, 160, 128 + 64, 64, 3), c(240, 320, 64 + 64, 32, 3),
          c(480, 640, 32 + 3, 32, 3) + c(480, 640, 32, 20, 1)]
    return g


METRICS = ["gpu__time_duration.sum", "sm__inst_executed_pipe_tensor_subpipe_hmma.avg.pct_of_peak_sustained_active",
           "sm__pipe_tensor_subpipe_hmma_cycles_active.avg.pct_of_peak_sustained_elapsed",
           "lts__throughput.avg.pct_of_peak_sustained_elapsed", "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed",
           "dram__bytes_read.sum", "dram__bytes_write.sum", "launch__registers_per_thread", "launch__grid_size",
           "sm__throughput.avg.pct_of_peak_sustained_elapsed"]


def raw(rep):
    out = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(out.splitlines()))
    h, units = rows[0], rows[1]
    return h, units, rows[2:]


def to_unit(v, unit, want):
    v = float(v.replace(",", ""))
    scale = {"ns": 1e-3, "us": 1.0, "ms": 1e3, "s": 1e6, "byte": 1e-6, "Kbyte": 1e-3, "Mbyte": 1.0, "Gbyte": 1e3}
    return v * scale.get(unit, 1.0) if want in ("us", "MB") else v


def conv(rep, md, js, batch=16):
    h, units, rows = raw(rep)
    col = {c: i for i, c in enumerate(h)}
    tens = [c for c in h if "tensor" in c and "pct" in c]
    gm = _gmac()
    lines = ["# ncu --set full, all 25 tensor-core conv launches (stem .. convraw.0 + fused head) of one bench step (batch 16, 480x640)", "",
             "`ncu --profile-from-start off --set full --clock-control none --import-source on -k "
             "regex:\"k_conv_tap|k_conv_col\" -c 25 python benchmarks/profile_step.py 1`"
             " -> `python benchmarks/ncu_tables.py conv ...`", "",
             "Times are under the profiler (serialised, cold): use shares. TFLOP/s = 2*GMAC*16 / time.", "",
             "`tensor pipe %` = the MMA sub-pipe doing math (max of the sm__*tensor*pct metrics); `tc active %` = "
             "`sm__pipe_tc_cycles_active` (the tensor-core pipe occupied, operand fetch included); `tc smem %` = "
             "`l1tex__data_pipe_tc_wavefronts_mem_shared` (the MMAs' shared-memory operand reads as a share of the L1 "
             "data pipe): a narrow layer shows a busy pipe that mostly waits for its A operand.", "",
             "| layer | kernel | grid | us | TFLOP/s | tensor pipe % | tc active % | tc smem % | L2 % | DRAM % | DRAM read MB | DRAM write MB | regs |",
             "|---|---|---|---|---|---|---|---|---|---|---|---|---|"]
    tot_us = rd = wr = 0.0
    for i, r in enumerate(rows[:25]):
        name = r[col["Kernel Name"]]
        short = name.split("(")[0].split("::")[-1]
        us = to_unit(r[col["gpu__time_duration.sum"]], units[col["gpu__time_duration.sum"]], "us")
        rmb = to_unit(r[col["dram__bytes_read.sum"]], units[col["dram__bytes_read.sum"]], "MB")
        wmb = to_unit(r[col["dram__bytes_write.sum"]], units[col["dram__bytes_write.sum"]], "MB")
        def num(v):
            try:
                return float(v.replace(",", ""))
            except ValueError:
                return 0.0
        tp = max(num(r[col[c]]) for c in tens) if tens else float("nan")
        l2 = float(r[col["lts__throughput.avg.pct_of_peak_sustained_elapsed"]])
        dr = float(r[col["gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed"]])
        tf = 2 * gm[i] * batch * 1e9 / (us * 1e-6) / 1e12
        tca = num(r[col["sm__pipe_tc_cycles_active.avg.pct_of_peak_sustained_elapsed"]]) \
            if "sm__pipe_tc_cycles_active.avg.pct_of_peak_sustained_elapsed" in col else float("nan")
        tcs = num(r[col["l1tex__data_pipe_tc_wavefronts_mem_shared.sum.pct_of_peak_sustained_elapsed"]]) \
            if "l1tex__data_pipe_tc_wavefronts_mem_shared.sum.pct_of_peak_sustained_elapsed" in col else float("nan")
        lines.append(f"| {LAYERS[i]} | `{short}` | {r[col['launch__grid_size']]} | {us:.1f} | {tf:.0f} | {tp:.1f} | {tca:.1f} | {tcs:.1f} | "
                     f"{l2:.1f} | {dr:.1f} | {rmb:.1f} | {wmb:.1f} | {r[col['launch__registers_per_thread']]} |")
        tot_us += us
        rd += rmb
        wr += wmb
    lines += ["", f"Totals: {tot_us:.1f} us, DRAM read {rd:.1f} + write {wr:.1f} MB per step."]
    open(md, "w").write("\n".join(lines) + "\n")
    json.dump({"what": "dram__bytes_read.sum + dram__bytes_write.sum summed over the 25 tensor-core conv launches of one "
                       "bench step (batch 16), ncu --set full",
               "dram_read_mb": round(rd, 1), "dram_write_mb": round(wr, 1), "bytes_per_step": int((rd + wr) * 1e6),
               "source": md}, open(js, "w"), indent=1)
    print("\n".join(lines[-3:]))


VOTE_METRICS = ["launch__grid_size", "launch__block_size", "gpu__time_duration.sum", "dram__bytes_read.sum",
                "dram__bytes_write.sum", "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed",
                "sm__throughput.avg.pct_of_peak_sustained_elapsed", "smsp__issue_active.avg.pct_of_peak_sustained_active",
                "sm__inst_executed_pipe_fma.avg.pct_of_peak_sustained_active",
                "sm__inst_executed_pipe_alu.avg.pct_of_peak_sustained_active",
                "sm__warps_active.avg.pct_of_peak_sustained_active", "launch__registers_per_thread",
                "launch__occupancy_limit_shared_mem", "launch__occupancy_limit_registers", "smsp__inst_executed.sum",
                "sm__cycles_elapsed.avg.per_second"]


VOTE_METRICS += ["sm__pipe_fma_cycles_active.avg.pct_of_peak_sustained_active",
                 "sm__inst_executed_pipe_lsu.avg.pct_of_peak_sustained_active",
                 "smsp__average_warps_issue_stalled_math_pipe_throttle_per_issue_active.ratio",
                 "smsp__average_warps_issue_stalled_wait_per_issue_active.ratio",
                 "smsp__average_warps_issue_stalled_long_scoreboard_per_issue_active.ratio",
                 "smsp__average_warps_issue_stalled_barrier_per_issue_active.ratio"]


def vote(rep, md, bench_json=None, hn=256):
    h, units, rows = raw(rep)
    col = {c: i for i, c in enumerate(h)}
    r = rows[0]
    fg, k = 20000.0, 9
    tests = int(16 * fg * k * hn)
    if bench_json:
        rv = json.load(open(bench_json))["roofline_vote"]
        fg = rv["fg_px_per_image"]
        tests = int(16 * fg * k * hn)                       # the kernel's own tests (the refit's +1 vote is k_refit's)
    if hn == 256:
        head = [f"# ncu --set full, k_vote3 inside one bench step (16 images x ~{fg:.0f} px, {hn} hyp, K={k})", "",
                "`ncu --profile-from-start off --set full --clock-control none --import-source on -k regex:k_vote3 -c 1 python "
                "benchmarks/profile_step.py 1` -> `python benchmarks/ncu_tables.py vote ...`", ""]
    else:
        head = [f"# ncu --set full, k_vote3 of the config-4 voting layer (16 images x {fg:.0f} px, 256 + 4096 hyp in one launch, K={k})",
                "", "`SUST_FIELD=planted SUST_SKIP_BURST=1 ncu --set full --clock-control none --import-source on -k regex:k_vote3 "
                "--launch-skip 6 -c 1 python benchmarks/vote_sustained.py` -> `python benchmarks/ncu_tables.py vote4 ...`", ""]
    lines = head + [
        f"Kernel: `{r[col['Kernel Name']][:100]}`", "", "| metric | value | unit |", "|---|---|---|"]
    for m in VOTE_METRICS + ["sm__pipe_alu_cycles_active.avg.pct_of_peak_sustained_active"]:
        if m in col:
            lines.append(f"| {m} | {r[col[m]]} | {units[col[m]]} |")
    inst = float(r[col["smsp__inst_executed.sum"]].replace(",", ""))
    us = to_unit(r[col["gpu__time_duration.sum"]], units[col["gpu__time_duration.sum"]], "us")
    rd = to_unit(r[col["dram__bytes_read.sum"]], units[col["dram__bytes_read.sum"]], "MB")
    wr = to_unit(r[col["dram__bytes_write.sum"]], units[col["dram__bytes_write.sum"]], "MB")
    alg = 16 * (fg * 4 + fg * k * 8 + hn * k * 8 + hn * k * 4) / 1e6        # pixel list + direct lists + hypotheses + counts
    lines += ["", f"Tests in this launch: 16 x ~{fg:.0f} px x {k} kp x {hn} hyp = {tests / 1e6:.0f} M -> "
                  f"{inst * 32 / tests:.2f} warp-instructions per 32 tests (all kernel phases included), "
                  f"{tests / (us * 1e-6) / 1e12:.2f}e12 tests/s under the profiler.",
              f"The kernel's algorithmic HBM bytes (compact pixel list 4 B/px + direct lists 8 B/px/keypoint + hypotheses + "
              f"counts) = {alg:.1f} MB; measured DRAM read + write = {rd + wr:.1f} MB = {(rd + wr) / alg:.2f}x "
              "(round 1, gathering sectors from the NCHW field per keypoint: 313 MB = 4.9x its 62.5 MB).",
              "It is FP32-pipe bound (FMA-pipe cycles and issue-active above), not HBM bound: DESIGN.md section 3."]
    open(md, "w").write("\n".join(lines) + "\n")
    print("\n".join(lines[6:]))


def launch_list(csvf, md, steps=2):
    rows = [r for r in csv.reader(open(csvf)) if len(r) > 5]
    h = rows[0]
    ik, iv, iu = h.index("Kernel Name"), h.index("Metric Value"), h.index("Metric Unit")
    agg = {}
    for r in rows[1:]:
        try:
            v = float(r[iv].replace(",", ""))
        except ValueError:
            continue
        v *= {"ns": 1e-3, "us": 1.0, "ms": 1e3}.get(r[iu], 1.0)
        a = agg.setdefault(r[ik][:72], [0, 0.0])
        a[0] += 1
        a[1] += v
    tot = sum(a[1] for a in agg.values())
    lines = [f"# ncu launch list (gpu__time_duration.sum), {steps} bench steps (batch 16)", "",
             "`ncu --profile-from-start off --metrics gpu__time_duration.sum --clock-control none --csv python "
             f"benchmarks/profile_step.py {steps}` -> `python benchmarks/ncu_tables.py list ...`", "",
             f"Total {tot / 1e3:.3f} ms for {steps} steps (cold, serialised: compare shares).", "",
             "| kernel | launches | total us | share |", "|---|---|---|---|"]
    for k, (n, v) in sorted(agg.items(), key=lambda x: -x[1][1]):
        lines.append(f"| `{k}` | {n} | {v:.1f} | {100 * v / tot:.1f}% |")
    open(md, "w").write("\n".join(lines) + "\n")
    print("\n".join(lines[4:12]))


def top(rep, kid, n=16):
    out = subprocess.run(f"ncu -i {rep} --page source --csv --print-source cuda,sass --kernel-id :::{kid}", shell=True,
                         capture_output=True, text=True).stdout
    rows = list(csv.reader(out.splitlines()))
    res, cur, hdr, name = [], None, None, ""
    for r in rows:
        if len(r) == 2 and r[0] == "File Path":
            cur, hdr = r[1], None
            continue
        if len(r) == 2 and r[0] == "Function Name":
            name = r[1]
            continue
        if r and r[0] == "Line No":
            hdr = r
            isamp = hdr.index("# Samples")
            continue
        if cur and hdr and len(r) == len(hdr) and r[0].isdigit() and r[2] == "-":
            sm = int(r[isamp]) if r[isamp].isdigit() else 0
            if sm:
                res.append((sm, cur.split("/")[-1], r[0], r[1].strip()[:100]))
    tot = sum(x[0] for x in res)
    print(f"--- kernel {kid} {name[:90]}: {tot} samples")
    for sm, f, ln, src in sorted(res, reverse=True)[:n]:
        print(f"{100 * sm / tot:5.1f}% {f}:{ln:>4} {src}")


def stalls(rep, label):
    """Markdown: key throughput metrics of the (single) captured kernel + where the warp-stall samples fall,
    per block of 100 SASS instructions (ncu --set full --import-source on)."""
    h, units, rows = raw(rep)
    col = {c: i for i, c in enumerate(h)}
    r = rows[0]
    keys = ["gpu__time_duration.sum", "launch__registers_per_thread", "launch__shared_mem_per_block_dynamic",
            "launch__occupancy_limit_shared_mem", "launch__occupancy_limit_registers",
            "sm__warps_active.avg.pct_of_peak_sustained_active", "sm__pipe_tc_cycles_active.avg.pct_of_peak_sustained_elapsed",
            "l1tex__data_pipe_tc_wavefronts_mem_shared.sum.pct_of_peak_sustained_elapsed",
            "l1tex__data_pipe_lsu_wavefronts.sum.pct_of_peak_sustained_elapsed",
            "smsp__issue_active.avg.pct_of_peak_sustained_active", "sm__inst_executed.sum",
            "lts__throughput.avg.pct_of_peak_sustained_elapsed", "dram__bytes_read.sum", "dram__bytes_write.sum",
            "l1tex__t_requests_pipe_lsu_mem_local_op_st.sum", "l1tex__t_requests_pipe_lsu_mem_local_op_ld.sum"]
    print(f"### {label}\n\n`{r[col['Kernel Name']][:70]}`\n\n| metric | value |\n|---|---|")
    for k in keys:
        if k in col:
            print(f"| `{k}` | {r[col[k]]} {units[col[k]]} |")
    out = subprocess.run(["ncu", "-i", rep, "--page", "source", "--csv"], capture_output=True, text=True).stdout
    srows = list(csv.reader(out.splitlines()))
    sh, data = srows[1], srows[2:]
    isamp, iexe = sh.index("# Samples"), sh.index("Instructions Executed")
    st = [i for i, c in enumerate(sh) if c.startswith("stall_") and "Not Issued" not in c]
    tot = sum(int(x[isamp]) for x in data)
    print(f"\nWarp-stall samples: {tot} over {len(data)} SASS instructions; blocks of 100 instructions holding >= 1 %:\n")
    print("| SASS index | samples | % | warp-instr. executed per (tile, warp) | top stall reasons | first instruction |\n|---|---|---|---|---|---|")
    for k in range(0, len(data), 100):
        seg = data[k:k + 100]
        sm = sum(int(x[isamp]) for x in seg)
        if sm < 0.01 * tot:
            continue
        ex = sum(int(x[iexe]) for x in seg) / 153600.0
        agg = {}
        for x in seg:
            for i in st:
                if x[i].isdigit():
                    agg[sh[i][6:]] = agg.get(sh[i][6:], 0) + int(x[i])
        top = ", ".join(f"{n} {v}" for n, v in sorted(agg.items(), key=lambda z: -z[1])[:3])
        print(f"| {k} | {sm} | {100 * sm / tot:.1f} | {ex:.0f} | {top} | `{seg[0][1].strip()[:38]}` |")
    print()


if __name__ == "__main__":
    cmd = sys.argv[1]
    if cmd == "conv":
        conv(sys.argv[2], sys.argv[3], sys.argv[4])
    elif cmd == "list":
        launch_list(sys.argv[2], sys.argv[3])
    elif cmd == "vote":
        vote(sys.argv[2], sys.argv[3], sys.argv[4] if len(sys.argv) > 4 else None)
    elif cmd == "vote4":
        vote(sys.argv[2], sys.argv[3], None, hn=4352)
    elif cmd == "stalls":
        stalls(sys.argv[2], sys.argv[3])
    elif cmd == "top":
        top(sys.argv[2], int(sys.argv[3]), int(sys.argv[4]) if len(sys.argv) > 4 else 16)
