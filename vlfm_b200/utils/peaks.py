"""Peak rates that roofline fractions are taken against (bench.py, scripts/bench_full_step.py)."""
from __future__ import annotations

import json
import os

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
# NVIDIA's data-sheet figures for the H100 SXM at 700 W: HBM3 3.35 TB/s, dense fp16/bf16 989 TFLOP/s
DATA_SHEET = {"hbm_gbs": 3350.0, "bf16_tflops": 989.0}


def peaks():
    """(rates, source): MEASURED_PEAKS.json at the repository root when someone measured the card, else the data sheet."""
    try:
        with open(os.path.join(ROOT, "MEASURED_PEAKS.json")) as fh:
            return json.load(fh), "measured"
    except Exception:
        return dict(DATA_SHEET), "H100 SXM data sheet"
