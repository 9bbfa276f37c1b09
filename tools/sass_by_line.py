#!/usr/bin/env python
"""Joins an ncu `--page source --csv` export (per-SASS-instruction counters) with `nvdisasm -g` line info of the same cubin:
instructions executed and stall samples per SOURCE LINE of a kernel.
usage: sass_by_line.py <ncu_source.csv> <nvdisasm.sass> <kernel name substring> [capture index] [top N]"""
import collections
import csv
import re
import sys


def load_ncu(path, kernel_sub, which):
    rows = list(csv.reader(open(path)))
    starts = [i for i, r in enumerate(rows) if r and r[0] == "Kernel Name"]
    blocks = []
    for k, s in enumerate(starts):
        e = starts[k + 1] if k + 1 < len(starts) else len(rows)
        if kernel_sub in rows[s][1]:
            blocks.append(rows[s:e])
    blk = blocks[which]
    hdr = blk[1]; ix = {h: i for i, h in enumerate(hdr)}
    out = []
    base = None
    for r in blk[2:]:
        try:
            addr = int(r[ix["Address"]], 16)
        except Exception:
            continue
        if base is None:
            base = addr
        out.append((addr - base, r[ix["Source"]].strip(), int(r[ix["Instructions Executed"]] or 0), int(r[ix["# Samples"]] or 0),
                    float(r[ix["Avg. Threads Executed"]] or 0)))
    return out


def load_lines(path, mangled_sub):
    """offset -> (file, line, inline chain) for the function whose section name contains mangled_sub"""
    m = {}
    cur = None; active = False
    for ln in open(path, errors="replace"):
        if ln.startswith(".text."):
            active = mangled_sub in ln
            continue
        if not active:
            continue
        mm = re.match(r'\s*//## File "([^"]+)", line (\d+)(.*)', ln)
        if mm:
            cur = (mm.group(1).split("/")[-1], int(mm.group(2)))
            continue
        mm = re.match(r"\s*/\*([0-9a-f]{4,})\*/\s+(.*)", ln)
        if mm and cur:
            m[int(mm.group(1), 16)] = cur
    return m


def main():
    ncu_csv, sass, ksub = sys.argv[1:4]
    which = int(sys.argv[4]) if len(sys.argv) > 4 else -1
    top = int(sys.argv[5]) if len(sys.argv) > 5 else 40
    mangled = {"pair_kernel": "pair11pair_kernel", "step_kernel<(int)2, (int)3>": "unrolled11step_kernelILi2ELi3E"}.get(ksub, ksub)
    inst = load_ncu(ncu_csv, ksub, which)
    lines = load_lines(sass, mangled)
    per = collections.defaultdict(lambda: [0, 0, 0.0])
    tot = samp = 0
    miss = 0
    for off, src, ie, s, thr in inst:
        key = lines.get(off)
        if key is None:
            miss += ie; key = ("?", 0)
        per[key][0] += ie; per[key][1] += s; per[key][2] += ie * thr
        tot += ie; samp += s
    print(f"total warp-instr {tot}  samples {samp}  unmapped {miss}")
    for key, (ie, s, thr) in sorted(per.items(), key=lambda kv: -kv[1][0])[:top]:
        print(f"{key[0]:18s} {key[1]:5d}  inst {ie:9d} {100 * ie / tot:5.1f}%  samples {100 * s / max(samp, 1):5.1f}%  thr/inst {thr / max(ie, 1):4.1f}")


if __name__ == "__main__":
    main()
