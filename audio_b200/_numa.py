"""Bind the calling process to the CPU cores (and so, by first touch, the memory) of one GPU's NUMA node.

Pinned host buffers that feed a GPU over PCIe should live on the socket the GPU hangs off: with one
process per GPU and no binding, ``pin_memory()`` lands wherever the rank happened to be scheduled and
half the ranks of a two-socket, 8-GPU machine pull their waveforms across the inter-socket link.  No dependency beyond sysfs; a no-op when the topology cannot be read.
"""
from __future__ import annotations

import os
from typing import Optional, Set


def _parse_cpulist(text: str) -> Set[int]:
    cpus: Set[int] = set()
    for part in text.strip().split(","):
        if not part:
            continue
        if "-" in part:
            lo, hi = part.split("-")
            cpus.update(range(int(lo), int(hi) + 1))
        else:
            cpus.add(int(part))
    return cpus


def gpu_numa_node(device_index: int) -> Optional[int]:
    """NUMA node of the PCI device behind ``cuda:<device_index>`` (None if unknown)."""
    try:
        import torch

        p = torch.cuda.get_device_properties(device_index)
        bdf = f"{p.pci_domain_id:04x}:{p.pci_bus_id:02x}:{p.pci_device_id:02x}.0"
        with open(f"/sys/bus/pci/devices/{bdf}/numa_node") as fh:
            node = int(fh.read().strip())
        return node if node >= 0 else None
    except Exception:
        return None


def bind_to_gpu(device_index: int, max_cpus: Optional[int] = None) -> dict:
    """``sched_setaffinity`` to the cores of the GPU's NUMA node (intersected with the current mask).

    Returns what was done: ``{"node": n, "cpus": count}`` or ``{"node": None, ...}`` when nothing changed.
    Call it BEFORE allocating pinned memory so the pages are first-touched on that node.
    """
    info = {"node": None, "cpus": len(os.sched_getaffinity(0)) if hasattr(os, "sched_getaffinity") else None}
    node = gpu_numa_node(device_index)
    if node is None or not hasattr(os, "sched_setaffinity"):
        return info
    try:
        with open(f"/sys/devices/system/node/node{node}/cpulist") as fh:
            cpus = _parse_cpulist(fh.read())
        cpus &= os.sched_getaffinity(0)
        if not cpus:
            return info
        if max_cpus is not None and len(cpus) > max_cpus:
            cpus = set(sorted(cpus)[:max_cpus])
        os.sched_setaffinity(0, cpus)
        info.update(node=node, cpus=len(cpus))
    except Exception:
        pass
    return info
