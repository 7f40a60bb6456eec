"""SASS report of the RANK / MTFT inverse step for blocks of at most 16 MiB (sbrt_inverse_multi_kernel, kanzi-go_b200/csrc/kz_sbrt.cu).

Cross-compiles kz_sbrt.cu for sm_90a with the library's flags (no GPU needed), disassembles it with cuobjdump and, for both instances
(RANK and MTFT), finds the fully unrolled round of 32 ranks: the loop whose body holds 32 CTA barriers. It prints the instructions of that
loop body per rank and warp (barrier, loads of the next round and output stores included) with the opcode mix, and the totals of the
whole function (set-up and tail loop included). With one warp per scheduler nothing hides a step's latency, and the chain's time follows
this count (DESIGN.md §4.3).

    python tools/sass_rank_inverse.py [--src kanzi-go_b200/csrc/kz_sbrt.cu] [--json]
"""
import argparse
import collections
import json
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "kanzi-go_b200", "csrc", "kz_sbrt.cu")
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17"]  # kanzi-go_b200/build.py, without the link
INSTANCES = (("RANK", "_ZN2kz25sbrt_inverse_multi_kernelILb1E"), ("MTFT", "_ZN2kz25sbrt_inverse_multi_kernelILb0E"))
ROUND = 32  # ranks per unrolled round

INSN = re.compile(r"/\*([0-9a-f]{4,})\*/\s+(@!?U?P[T0-9]+\s+)?([A-Z0-9_.]+)([^;]*);")


def disassemble(src):
    with tempfile.TemporaryDirectory() as tmp:
        cubin = os.path.join(tmp, "kz_sbrt.cubin")
        subprocess.run(["nvcc", "-cubin"] + FLAGS + [src, "-o", cubin], check=True)
        return subprocess.run(["cuobjdump", "-sass", cubin], check=True, capture_output=True, text=True).stdout


def functions(sass):
    """name -> [(address, opcode, operands)] in address order"""
    out, name = {}, None
    for line in sass.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            name = m.group(1)
            out[name] = []
            continue
        m = INSN.search(line)
        if m and name:
            out[name].append((int(m.group(1), 16), m.group(3), m.group(4).strip()))
    return out


def base_op(op):
    return op.split(".")[0]


def mix(insns):
    return collections.Counter(base_op(op) for _, op, _ in insns if op != "NOP")


def round_loop(insns):
    """the body of the loop (backward branch) that holds ROUND barriers"""
    addr = [a for a, _, _ in insns]
    for k, (a, op, args) in enumerate(insns):
        if base_op(op) != "BRA":
            continue
        m = re.match(r"(0x[0-9a-f]+)", args)
        if not m or int(m.group(1), 16) >= a:
            continue
        body = insns[addr.index(int(m.group(1), 16)): k + 1]
        if sum(base_op(op) == "BAR" for _, op, _ in body) == ROUND:
            return body
    raise SystemExit("no loop with %d barriers found: the round of %d ranks is not fully unrolled" % (ROUND, ROUND))


def report(sass):
    funcs = functions(sass)
    res = {}
    for label, prefix in INSTANCES:
        names = [f for f in funcs if f.startswith(prefix)]
        if len(names) != 1:
            raise SystemExit("%s instance of sbrt_inverse_multi_kernel not found" % label)
        insns = funcs[names[0]]
        body = round_loop(insns)
        m = mix(body)
        res[label] = dict(per_rank=sum(m.values()) / ROUND, round=sum(m.values()), mix={k: v / ROUND for k, v in m.most_common()},
                          function=sum(mix(insns).values()), function_mix=dict(mix(insns).most_common()))
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--src", default=SRC)
    ap.add_argument("--json", action="store_true")
    a = ap.parse_args()
    res = report(disassemble(a.src))
    if a.json:
        print(json.dumps(res, indent=1))
        return
    for label, r in res.items():
        print("%s: %.2f instructions per rank and warp (%d in the unrolled round of %d ranks, barrier included); whole function %d"
              % (label, r["per_rank"], r["round"], ROUND, r["function"]))
        print("  per rank: " + ", ".join("%s %.2f" % (k, v) for k, v in r["mix"].items()))
        fm = r["function_mix"]
        print("  function: " + ", ".join("%s %d" % (k, fm.get(k, 0)) for k in ("SHFL", "ISETP", "SEL", "LDS", "STS", "BAR", "PRMT")))


if __name__ == "__main__":
    sys.exit(main())
