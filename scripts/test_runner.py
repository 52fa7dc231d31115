"""Run the CPU test-suite and keep a log under $BEE2BEE_HOME (parity: /root/reference/scripts/test_runner.py, which only
import-smokes its test modules; this one actually runs them through pytest).

    python scripts/test_runner.py            # -m "not gpu"
    python scripts/test_runner.py --gpu      # kernel / model / multi-GPU tiers on a H100 host
"""
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main() -> int:
    from bee2bee_b200.utils import data_file

    marker = "gpu" if "--gpu" in sys.argv else "not gpu"
    log_path = str(data_file("test.log"))
    t0 = time.time()
    res = subprocess.run([sys.executable, "-m", "pytest", os.path.join(ROOT, "tests"), "-q", "-m", marker, "-p", "no:cacheprovider"],
                         cwd=ROOT, capture_output=True, text=True)
    with open(log_path, "a") as f:
        f.write(f"==== {time.strftime('%Y-%m-%d %H:%M:%S')} -m '{marker}' exit {res.returncode} in {time.time() - t0:.1f}s\n")
        f.write(res.stdout[-20000:] + res.stderr[-5000:] + "\n")
    print(res.stdout.strip().splitlines()[-1] if res.stdout.strip() else res.stderr[-500:])
    print(f"log: {log_path}")
    return res.returncode


if __name__ == "__main__":
    raise SystemExit(main())
