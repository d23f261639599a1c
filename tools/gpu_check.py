"""Run the GPU kernel tests group by group in isolated subprocesses (a trapped kernel poisons its CUDA context),
each under its own timeout; logs go to tools_out/. Usage: python tools/gpu_check.py [group ...]"""
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "tools_out")
os.makedirs(OUT, exist_ok=True)

GROUPS = [
    ("tests/test_kernels_gpu.py", "test_gemm_plain"),
    ("tests/test_kernels_gpu.py", "test_gemm_epilogues"),
    ("tests/test_kernels_gpu.py", "test_gemm_geglu"),
    ("tests/test_kernels_gpu.py", "test_gemm_layernorm_fold"),
    ("tests/test_kernels_gpu.py", "test_attention_kv_split"),
    ("tests/test_kernels_gpu.py", "test_conv3x3"),
    ("tests/test_kernels_gpu.py", "test_attention"),
    ("tests/test_kernels_gpu.py", "norm"),
    ("tests/test_kernels_gpu.py", "test_linear_small or test_sinusoid or test_upsample or test_euler"),
]


def main():
    want = sys.argv[1:]
    summary = []
    for f, k in GROUPS:
        if want and not any(w in k for w in want):
            continue
        tag = k.split(" ")[0]
        log = os.path.join(OUT, f"check_{tag}.log")
        t0 = time.time()
        cmd = [sys.executable, "-m", "pytest", f, "-m", "gpu", "-k", k, "-q", "-s", "-p", "no:cacheprovider",
               "--timeout", "300"]
        try:
            r = subprocess.run(cmd, cwd=ROOT, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, timeout=900)
            rc, text = r.returncode, r.stdout.decode(errors="replace")
        except subprocess.TimeoutExpired as e:
            rc, text = -9, (e.stdout or b"").decode(errors="replace") + "\n[TIMEOUT]"
        with open(log, "w") as fh:
            fh.write(text)
        tail = [l for l in text.strip().splitlines() if l.strip()][-1:] or ["?"]
        summary.append(f"{tag}: rc={rc} {time.time() - t0:.0f}s :: {tail[0]}")
        print(summary[-1], flush=True)
        # show failures / error lines
        for l in text.splitlines():
            if ("Error" in l or "FAILED" in l or "out of tolerance" in l or "non-finite" in l) and len(l) < 400:
                print("    " + l)
    with open(os.path.join(OUT, "check_summary.txt"), "w") as fh:
        fh.write("\n".join(summary) + "\n")


if __name__ == "__main__":
    main()
