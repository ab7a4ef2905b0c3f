"""Prints a markdown table: per kernel of the shipped library, how often the SASS mnemonics that prove the
design claims occur (TMA bulk copies, pair-array sweep loads and FFMA, 128-bit reductions/stores, warp reductions, mbarriers).
    python tools/sass_counts.py [toypathtracer_b200/libtpt_b200.so] > sass_counts.md
tests/test_sass_claims.py imports kernel_counts() to pin the claims on every build."""
import re, subprocess, sys, collections

COLS = [("UBLKCP", r"\bUBLKCP"), ("LDS.128", r"\bLDS\.128"), ("FFMA", r"\bFFMA(\.[A-Z]+)*\s"), ("FFMA2", r"\bFFMA2"), ("FADD2", r"\bFADD2"), ("REDG.F32x4", r"\bREDG\.E\.ADD\.F32x4"),
        ("(C)REDUX", r"\bC?REDUX"), ("STG.128", r"\bSTG\.E(\.[A-Z0-9_]+)*\.128"), ("ATOMS", r"\bATOMS"), ("SYNCS", r"\bSYNCS"), ("MUFU", r"\bMUFU"),
        ("DFMA", r"\bDFMA"), ("LD.E (generic)", r"\bLD\.E"), ("BRX", r"\bBRX"), ("tensor", r"\b(HMMA|IMMA|DMMA|QMMA|UTCHMMA|UTCIMMA|UTCQMMA|UTCMMA|HGMMA)")]


def demangle(n):
    d = subprocess.run(["cu++filt", n], capture_output=True, text=True).stdout.strip() or n
    d = re.sub(r"\((int|bool|unsigned int)\)", "", d); d = re.sub(r"^(void )?tpt::", "", d)
    return re.sub(r"\(.*$", "", d)


def kernel_counts(lib):
    """[(demangled kernel name, instruction count, Counter of COLS names)] for every kernel in the library."""
    sass = subprocess.run(["cuobjdump", "-sass", lib], capture_output=True, text=True).stdout
    rows, cur, cnt, n = [], None, None, 0
    for line in sass.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            if cur: rows.append((demangle(cur), n, cnt))
            cur, cnt, n = m.group(1), collections.Counter(), 0
            continue
        if cur and re.match(r"\s+/\*[0-9a-f]{4,}\*/", line):
            n += 1
            for name, rx in COLS:
                if re.search(rx, line): cnt[name] += 1
    if cur: rows.append((demangle(cur), n, cnt))
    return rows


if __name__ == "__main__":
    lib = sys.argv[1] if len(sys.argv) > 1 else "toypathtracer_b200/libtpt_b200.so"
    print("# SASS evidence per kernel (`python tools/sass_counts.py`: cuobjdump -sass toypathtracer_b200/libtpt_b200.so, sm_90a only)\n")
    print("UBLKCP = TMA bulk copy (cp.async.bulk.shared::cluster.global); REDG.F32x4 = red.global.add.v4.f32; (C)REDUX = __reduce_min_sync;")
    print("FFMA = scalar FP32 FMA; FFMA2/FADD2 = packed f32x2 math (none on sm_90a); STG.128 = 128-bit global store (incl. .NA = L1::no_allocate);")
    print("SYNCS = mbarrier ops; DFMA = the glibc-faithful double-precision sinf/cosf/powf; LD.E = generic-address loads (0 in the 128-thread")
    print("queue/group instances: every scene section is addressed as shared memory); BRX = indirect branch (jump table); tensor = any")
    print("tensor-core opcode (none: no contraction on this path). tests/test_sass_claims.py asserts the load-bearing cells.\n")
    print("| kernel | instr | " + " | ".join(c for c, _ in COLS) + " |")
    print("|---|---|" + "---|" * len(COLS))
    for name, n, cnt in kernel_counts(lib):
        print(f"| `{name}` | {n} | " + " | ".join(str(cnt[c]) for c, _ in COLS) + " |")
