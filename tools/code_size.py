#!/usr/bin/env python
"""Developer aid: SASS size of rx_fused_split_kernel<5,5> with one warp role compiled out at a time."""
import os, re, shutil, subprocess, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "gen2_uhf_rfid_reader_b200", "csrc")
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-fmad=false", "-cubin"]
variants = {"full": None, "no workers": "if (role >= 2 && role < 2 + kSWWarps) {", "no chain": "} else if (role == 0) {",
            "no control": "} else if (role == 1) {", "no decoder": "DECODER"}
for name, pat in variants.items():
    d = "/tmp/sz_%d" % os.getpid()
    shutil.rmtree(d, ignore_errors=True)
    shutil.copytree(os.path.join(ROOT, "gen2_uhf_rfid_reader_b200"), os.path.join(d, "gen2_uhf_rfid_reader_b200"),
                    ignore=shutil.ignore_patterns("*.so", "__pycache__"))
    shutil.copytree(os.path.join(ROOT, "include"), os.path.join(d, "include"))
    f = os.path.join(d, "gen2_uhf_rfid_reader_b200", "csrc", "rx_fused_split.cuh")
    s = open(f).read()
    if pat == "DECODER":
        i = s.index("    // =========================================================== decoder")
        j = s.index("    PH_END(23)")
        s = s[:i] + s[j:]
    elif pat:
        assert pat in s
        s = s.replace(pat, pat.replace("role >= 2 && role < 2 + kSWWarps", "false").replace("role == 0", "false").replace("role == 1", "false"))
    open(f, "w").write(s)
    out = os.path.join(d, "k.cubin")
    subprocess.check_call(["nvcc"] + FLAGS + ["-o", out, os.path.join(d, "gen2_uhf_rfid_reader_b200", "csrc", "rfid_b200.cu")],
                          stderr=subprocess.DEVNULL)
    sass = subprocess.run(["cuobjdump", "-sass", out], capture_output=True, text=True).stdout
    cur, cnt = None, {}
    for line in sass.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = m.group(1)
        elif re.match(r"^\s+/\*[0-9a-f]+\*/\s+[A-Z@]", line) and cur:
            cnt[cur] = cnt.get(cur, 0) + 1
    k = [v for n, v in cnt.items() if "split_kernelILi5ELi5" in n][0]
    print("%-12s %6.1f KB" % (name, k * 16 / 1024))
    shutil.rmtree(d, ignore_errors=True)
