"""Black-box tuning of the N-tile cost model of the TMA conv kernel (conv_tma.cu: choose_bn): runs tools/layer_times.py once per
MITB_CM setting ("mode,epi_gelu,epi,fix,epi_reg") in a fresh process and prints the conv-class milliseconds per page of each."""
import json
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SETTINGS = sys.argv[1:] or ["1,225,350,600,450", "1,300,450,600,450", "1,150,250,600,450", "1,225,350,600,300", "1,225,350,600,600"]
for cm in SETTINGS:
    env = dict(os.environ, MITB_CM=cm)
    out = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "layer_times.py")], env=env, capture_output=True, text=True).stdout
    m = re.search(r"total ms ([0-9.]+)", out)
    tail = out.strip().splitlines()[-1] if out.strip() else "{}"
    try:
        conv = json.loads(tail).get("conv_tc", {}).get("ms")
    except Exception:
        conv = None
    print(f"MITB_CM={cm:16s} conv launches total ms {m.group(1) if m else '?':>8s}   conv_tc class ms {conv}")
    sys.stdout.flush()
