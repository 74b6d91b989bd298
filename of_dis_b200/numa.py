"""Host-side placement for the pinned staging buffers.

On a two-socket host a pinned buffer that lands on the socket remote from the GPU is
read over the inter-socket link: the H2D copy of a batch then runs at about half the
PCIe rate (tools/upload_timing.py measures both).
`bind_to_gpu_node(dev)` pins the calling thread to the CPUs of the GPU's NUMA node so that
buffers allocated (first-touched) afterwards are local; `unbind(prev)` restores the mask.
Pure sysfs + sched_setaffinity; does nothing when the topology cannot be read.
"""
from __future__ import annotations

import os
import subprocess


def _parse_cpulist(text: str) -> set[int]:
    cpus: set[int] = set()
    for part in text.strip().split(","):
        if not part:
            continue
        lo, _, hi = part.partition("-")
        cpus.update(range(int(lo), int(hi or lo) + 1))
    return cpus


def gpu_pci_bus_id(device: int) -> str | None:
    """'0000:1b:00.0'-style sysfs name of CUDA device `device` of this process."""
    try:
        import torch

        p = torch.cuda.get_device_properties(device)
        return "%04x:%02x:%02x.0" % (p.pci_domain_id, p.pci_bus_id, p.pci_device_id)
    except Exception:
        pass
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=pci.bus_id", "--format=csv,noheader", "-i", str(device)],
                             capture_output=True, text=True, timeout=10).stdout.strip().lower()
        dom, rest = out.split(":", 1)
        return dom[-4:] + ":" + rest
    except Exception:
        return None


def gpu_numa_cpus(device: int) -> tuple[int | None, set[int]]:
    bus = gpu_pci_bus_id(device)
    if not bus:
        return None, set()
    try:
        node = int(open("/sys/bus/pci/devices/%s/numa_node" % bus).read())
        if node < 0:
            return None, set()
        cpus = _parse_cpulist(open("/sys/devices/system/node/node%d/cpulist" % node).read())
        return node, cpus
    except (OSError, ValueError):
        return None, set()


def bind_to_gpu_node(device: int):
    """Returns (node, previous_mask); node is None when nothing was changed."""
    node, cpus = gpu_numa_cpus(device)
    try:
        prev = os.sched_getaffinity(0)
        want = cpus & prev
        if node is None or not want:
            return None, prev
        os.sched_setaffinity(0, want)
        return node, prev
    except (AttributeError, OSError):
        return None, None


def unbind(prev) -> None:
    if prev:
        try:
            os.sched_setaffinity(0, prev)
        except OSError:
            pass
