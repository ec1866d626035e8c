"""
Multi-GPU plumbing: one process per GPU (torchrun), reads sharded embarrassingly, result records gathered to the
writer rank (SURVEY.md 8(e)).  The alignments themselves never communicate; the only exchange step is the gather
of fixed-size 9 x int32 records (36 B per alignment) -- over NCCL/NVLink on the GPU box, over gloo in the CPU tests.
"""
import numpy as np


def shard_bounds(n_items, world_size):
    """Contiguous, balanced-by-count shard boundaries: int64[world_size + 1]."""
    base, rem = divmod(int(n_items), int(world_size))
    sizes = [base + (1 if r < rem else 0) for r in range(world_size)]
    return np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)


def shard_bounds_by_bases(seq_off, world_size):
    """Contiguous shard boundaries balanced on the sum of sequence lengths (full-read scans, SURVEY 8(e))."""
    seq_off = np.asarray(seq_off, dtype=np.int64)
    n = len(seq_off) - 1
    total = int(seq_off[-1] - seq_off[0])
    bounds = [0]
    for r in range(1, world_size):
        target = seq_off[0] + (total * r) // world_size
        k = int(np.searchsorted(seq_off, target, side='left'))
        bounds.append(min(max(k, bounds[-1]), n))
    bounds.append(n)
    return np.asarray(bounds, dtype=np.int64)


def gather_records(local, counts, dst=0, group=None):
    """
    Gather per-rank record tensors (int32[count_r, 9], on the device for NCCL or on the CPU for gloo) to `dst`.
    `counts` are the per-rank record counts (known to every rank from the shard bounds).  Returns the
    concatenated int32[sum(counts), 9] tensor on dst, None elsewhere.  One `gather` to the writer rank (every rank sends
    its shard once; ranks are padded to the largest shard so the collective has equal-size buffers).
    """
    import torch
    import torch.distributed as dist
    world = dist.get_world_size(group)
    rank = dist.get_rank(group)
    if world == 1:
        return local
    mx = int(max(counts))
    if local.shape[0] == mx:
        pad = local.contiguous()
    else:
        pad = torch.zeros((mx, local.shape[1]), dtype=local.dtype, device=local.device)
        pad[:local.shape[0]] = local
    bucket = [torch.empty_like(pad) for _ in range(world)] if rank == dst else None
    dist.gather(pad, bucket, dst=dst, group=group)
    if rank != dst:
        return None
    return torch.cat([bucket[r][:int(counts[r])] for r in range(world)], dim=0)


def _cpulist(text):
    cpus = []
    for part in text.strip().split(','):
        if not part:
            continue
        lo, _, hi = part.partition('-')
        cpus.extend(range(int(lo), int(hi or lo) + 1))
    return cpus


def bind_host_to_gpu(pci_bus_id, local_world=1, local_rank=0):
    """
    Pin this process to the CPU cores of the NUMA node its GPU hangs off (sysfs: /sys/bus/pci/devices/<bdf>/numa_node,
    /sys/devices/system/node/nodeK/cpulist), sharing the node's cores between the ranks whose GPUs sit on it.  Pinned
    host buffers allocated afterwards are first-touched on that node, so the rank's H2D / D2H copies and its host-side
    packing stay NUMA-local.
    Returns {'node': k, 'cpus': n} or None when the topology cannot be read (nothing is changed then).
    """
    import os
    try:
        bdf = pci_bus_id.lower()
        if len(bdf.split(':')[0]) == 8:          # CUDA prints an 8-digit domain, sysfs uses 4
            bdf = bdf[4:]
        with open('/sys/bus/pci/devices/%s/numa_node' % bdf) as f:
            node = int(f.read().strip())
        if node < 0:
            return None
        with open('/sys/devices/system/node/node%d/cpulist' % node) as f:
            cpus = _cpulist(f.read())
        allowed = sorted(set(cpus) & set(os.sched_getaffinity(0)))
        if not allowed:
            return None
        # ranks on the same node split its cores; the mapping rank -> node is not known across ranks without a
        # collective, so every rank takes the slice (local_rank mod ranks_per_node) of an even split
        nodes = len([d for d in os.listdir('/sys/devices/system/node') if d.startswith('node') and d[4:].isdigit()])
        per_node = max(1, (int(local_world) + nodes - 1) // max(nodes, 1))
        k = int(local_rank) % per_node
        share = allowed[k * len(allowed) // per_node:(k + 1) * len(allowed) // per_node] or allowed
        os.sched_setaffinity(0, share)
        return {'node': node, 'cpus': len(share)}
    except (OSError, ValueError):
        return None
