"""What every benchmark tool records beside its times: the card it ran on."""
import subprocess

import torch


def card(device_index):
    """{"gpu", "power_limit", "sm_clock_max"} of GPU device_index, from one read-only nvidia-smi query.  A time is only
    comparable with another taken at the same power limit and clock ceiling.  Without nvidia-smi the name comes from torch
    and the other two fields are "unavailable"."""
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader",
                            "-i", str(device_index)], capture_output=True, text=True)
        fields = [s.strip() for s in q.stdout.strip().split(",")] if q.returncode == 0 else []
    except OSError:
        fields = []
    if len(fields) == 3:
        return dict(zip(("gpu", "power_limit", "sm_clock_max"), fields))
    return {"gpu": torch.cuda.get_device_name(device_index), "power_limit": "unavailable", "sm_clock_max": "unavailable"}
