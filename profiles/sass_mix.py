#!/usr/bin/env python
"""Opcode histogram (SASS, sm_90a) of the hot kernels in liblitegs_b200.so -- static evidence next to ncu captures:
which pipes a kernel's instruction stream leans on, and that the Hopper forms it relies on are really in the binary
(LDGSTS = cp.async, UBLKCP = cp.async.bulk / TMA 1-D, REDG = fire-and-forget RED, REDUX, MUFU.EX2/RCP).
usage: python profiles/sass_mix.py > sass_mix.txt"""
import collections
import re
import subprocess
import sys

LIB = "litegs_b200/liblitegs_b200.so"
KERNELS = [("raster_forward_kernel<8,16> (default: cp.async staging)", r"raster_forward_kernelILi8ELi16ELb0ELb0E"),
           ("raster_backward_v2_kernel<8,16> (round-2 default: packed fp32 pairs, raw moments, cp.async staging)",
            r"raster_backward_v2_kernelILi8ELi16ELb0ELb0ELb0E"),
           ("raster_backward_kernel<8,16> (round-1 scalar kernel, LGS_BWD=v1: cp.async, shared-memory reduce)", r"raster_backward_kernelILi8ELi16ELb0ELb0ELb0ELb1E"),
           ("raster_forward_kernel<16,16> with cp.async.bulk staging", r"raster_forward_kernelILi16ELi16ELb0ELb1E"),
           ("project_forward_kernel<3,8,16>", r"project_forward_kernelILi3ELi8ELi16E"),
           ("project_backward_kernel<3>", r"project_backward_kernelILi3E"),
           ("emit_pairs_rec_kernel<8,16,u16>", r"emit_pairs_rec_kernelILi8ELi16EtE"),
           ("rs_scatter_kernel<u16,16>", r"rs_scatter_kernelItLi16E"),
           ("rs_hist_kernel<u16,16,vec>", r"rs_hist_kernelItLi16ELb1E"),
           ("tile_range_bsearch_kernel<u16>", r"tile_range_bsearch_kernelItE"),
           ("ssim_forward_kernel<L1,train>", r"ssim_forward_kernelILb1ELb1E"),
           ("ssim_backward_kernel<L1,uniform>", r"ssim_backward_kernelILb1ELb1E"),
           ("adam_dense_kernel<clear>", r"adam_dense_kernelILb1E"),
           ("nvls_allreduce_f32_kernel (opt-in own all-reduce over the NVSwitch multicast address)", r"nvls_allreduce_f32_kernel")]


def main():
    sass = subprocess.run(["cuobjdump", "-sass", LIB], capture_output=True, text=True).stdout
    blocks = re.split(r"\n\s*Function : ", sass)
    print("# opcode histograms from `cuobjdump -sass litegs_b200/liblitegs_b200.so` (whole kernel, all paths; counts are static)")
    for title, pat in KERNELS:
        body = next((b for b in blocks if re.match(r"\S*" + pat, b)), None)
        if body is None:
            print(f"\n== {title}: not found")
            continue
        ops = collections.Counter()
        for ln in body.splitlines():
            m = re.match(r"\s+/\*[0-9a-f]{4,5}\*/\s+(?:@!?U?P\w+\s+)?([A-Z][A-Z0-9_]*)((?:\.[A-Z0-9_]+)*)", ln)
            if m:
                op = m.group(1)
                if op in ("MUFU", "LDGSTS", "UBLKCP", "REDG", "RED", "REDUX", "ATOMS", "ATOMG", "LDS", "STS", "LDG", "STG", "SHFL", "VOTE", "MATCH"):
                    if op == "MUFU" and m.group(2):
                        op += "." + m.group(2).split(".")[1]          # MUFU.EX2 / MUFU.RCP / MUFU.RSQ ...
                ops[op] += 1
        total = sum(ops.values())
        print(f"\n== {title}: {total} instructions")
        print("   " + "  ".join(f"{k} {v}" for k, v in ops.most_common(22)))
        # the forms that prove what the kernel is built on, wherever they rank
        marks = ("LDGSTS", "UBLKCP", "SYNCS", "REDG", "RED", "REDUX", "ATOMS", "ATOMG", "MUFU.EX2", "MUFU.RCP",
                 "MATCH", "SHFL", "VOTE", "LDGMC", "STGMC", "MULTIMEM")
        seen = [f"{k} {ops[k]}" for k in marks if ops.get(k)]
        if seen:
            print("   marks: " + "  ".join(seen))


if __name__ == "__main__":
    sys.exit(main())
