"""Summarise an `ncu --set full` report (.ncu-rep) into a markdown table: per kernel the duration, DRAM traffic, tensor-pipe /
shared-memory-operand utilisation and the top warp-stall sites.  Usage: python tools/ncu_summary.py report.ncu-rep [...] > summary.md
(runs `ncu -i` locally; no GPU needed)."""
import csv, io, subprocess, sys, collections

KEYS = [
    ("gpu__time_duration.sum", "duration"),
    ("sm__cycles_elapsed.avg", "SM cycles"),
    ("dram__bytes_read.sum", "DRAM read"),
    ("dram__bytes_write.sum", "DRAM write"),
    ("launch__grid_size", "grid"),
    ("launch__block_size", "block"),
    ("launch__registers_per_thread", "regs/thread"),
    ("launch__shared_mem_per_block_dynamic", "dyn smem/block"),
    ("sm__pipe_tc_cycles_active.avg.pct_of_peak_sustained_elapsed", "tensor pipe (tc) cycles active"),
    ("sm__pipe_tensor_op_gmma_cycles_active.avg.pct_of_peak_sustained_elapsed", "wgmma pipe cycles active"),
    ("l1tex__data_pipe_tc_wavefronts_mem_shared.sum.pct_of_peak_sustained_elapsed", "tensor-core smem operand wavefronts vs peak"),
    ("sm__inst_executed.avg.pct_of_peak_sustained_elapsed", "instruction issue vs peak"),
    ("lts__t_sector_hit_rate.pct", "L2 hit rate"),
    ("lts__throughput.avg.pct_of_peak_sustained_elapsed", "L2 throughput vs peak"),
    ("l1tex__data_bank_conflicts_pipe_lsu_mem_shared_op_ldgsts.sum", "cp.async smem bank conflicts"),
]


def ncu_csv(rep, page, extra=()):
    out = subprocess.run(["ncu", "-i", rep, "--page", page, "--csv", *extra], capture_output=True, text=True).stdout
    return list(csv.reader(io.StringIO(out)))


def main():
    for rep in sys.argv[1:]:
        rows = ncu_csv(rep, "raw")
        hdr, units = rows[0], rows[1]
        print("## `%s`\n" % rep.split("/")[-1])
        # the source page holds one table per profiled launch, each introduced by a "Kernel Name" row
        sections, cur = [], None
        for x in ncu_csv(rep, "source"):
            if x and x[0] == "Kernel Name":
                cur = [x]
                sections.append(cur)
            elif cur is not None:
                cur.append(x)
        kidx = 0
        for r in rows[2:]:
            name = r[hdr.index("Kernel Name")]
            print("### `%s`\n" % name[:110])
            print("| metric | value |\n|---|---|")
            for k, label in KEYS:
                if k in hdr:
                    v = r[hdr.index(k)]
                    try:
                        v = "%.4g" % float(v)
                    except ValueError:
                        pass
                    print("| %s (`%s`) | %s %s |" % (label, k, v, units[hdr.index(k)]))
            print()
            # match the source table of this launch by kernel name (template arguments included)
            import re
            def fn(n):
                m = re.search(r"(\w+<[^>]*>|\w+)\(", n.replace("(int)", "").replace(" ", ""))
                return m.group(1) if m else n
            key = fn(name)
            src = []
            for si, sec in enumerate(sections):
                if sec is not None and len(sec[0]) > 1 and fn(sec[0][1]) == key:
                    src, sections[si] = sec, None
                    break
            if len(src) < 3:
                continue
            h2 = src[1]
            data = [x for x in src[2:] if len(x) == len(h2) and x[h2.index('# Samples')].isdigit()]
            iS, iSrc = h2.index("# Samples"), h2.index("Source")
            stall = [i for i, h in enumerate(h2) if h.startswith("stall_") and "Not Issued" not in h]
            tot = sum(int(x[iS]) for x in data) or 1
            agg = collections.Counter()
            for x in data:
                for i in stall:
                    agg[h2[i]] += int(x[i])
            print("Warp-state samples (all warps): " + ", ".join("%s %.0f%%" % (k.replace("stall_", ""), 100.0 * v / tot) for k, v in agg.most_common(6)))
            print("\nHottest instructions (share of samples, dominant stall):\n")
            for x in sorted(data, key=lambda x: -int(x[iS]))[:6]:
                st = max(((int(x[i]), h2[i]) for i in stall))
                print("* %.1f%% `%s` — %s" % (100.0 * int(x[iS]) / tot, x[iSrc].strip()[:70], st[1].replace("stall_", "")))
            print()


if __name__ == "__main__":
    main()
