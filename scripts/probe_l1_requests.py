"""Build and run scripts/probe_l1_requests.cu (compiled into a temporary directory) and print its table with the
card's name, power limit and SM clock limit beside it.

    python scripts/probe_l1_requests.py
"""
import os
import subprocess
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))

from pumiumtally_b200 import build as pbuild  # noqa: E402


def main():
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True)
    print("card:", card.stdout.strip() or card.stderr.strip(), flush=True)
    with tempfile.TemporaryDirectory() as tmp:
        exe = os.path.join(tmp, "probe_l1_requests")
        subprocess.run([pbuild._nvcc(), "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17",
                        os.path.join(HERE, "probe_l1_requests.cu"), "-o", exe], check=True)
        subprocess.run([exe], check=True)


if __name__ == "__main__":
    main()
