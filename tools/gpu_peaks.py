"""Device facts the measurement tools divide by, read from the card they run on rather than assumed."""
import json
import os
import subprocess

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
H100_SXM_HBM_GBS = 3350.0          # NVIDIA data sheet, H100 SXM (a figure for a 700 W card, not a measurement)


def sm_count(device: int = 0) -> int:
    return torch.cuda.get_device_properties(device).multi_processor_count


def max_sm_clock_hz(device: int = 0) -> float:
    """The card's maximum SM clock as nvidia-smi reports it (a power-limited card may run below it under load)."""
    out = subprocess.run(["nvidia-smi", "-i", str(device), "--query-gpu=clocks.max.sm", "--format=csv,noheader,nounits"],
                         capture_output=True, text=True, check=True).stdout
    return float(out.strip().splitlines()[0]) * 1e6


def hbm_peak_gbs():
    """(peak GB/s, where it comes from): MEASURED_PEAKS.json's hbm_gbs when the file exists, else the H100 SXM data sheet."""
    try:
        return float(json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))["hbm_gbs"]), "measured (MEASURED_PEAKS.json)"
    except (OSError, KeyError, ValueError):
        return H100_SXM_HBM_GBS, "H100 SXM data sheet, not measured"
