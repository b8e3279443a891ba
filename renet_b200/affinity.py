"""CPU placement of one-process-per-GPU jobs on a multi-socket host.

On a typical two-socket 8-GPU server GPUs 0-3 hang off NUMA node 0 and GPUs 4-7 off node 1.  The end-to-end path of this repo is
host-driven (batch planning in loader threads, one consumer thread issuing CUDA calls), so eight ranks whose threads
float over both sockets -- and over each other's cores -- lose more than half of their throughput (round-1 SCALE:
e2e efficiency 0.43 at N=8).  ``pin_rank`` restricts the calling process (and every thread it creates afterwards) to
its GPU's NUMA node, and inside the node to this rank's own share of the cores the container may use.
"""
import os


def _parse_cpulist(txt):
    out = []
    for part in txt.strip().split(','):
        if not part:
            continue
        if '-' in part:
            a, b = part.split('-')
            out.extend(range(int(a), int(b) + 1))
        else:
            out.append(int(part))
    return out


def gpu_numa_node(local_rank):
    """NUMA node of the GPU this rank drives, or None when the platform does not say."""
    bus = None
    try:
        import pynvml
        pynvml.nvmlInit()
        vis = os.environ.get('CUDA_VISIBLE_DEVICES')
        idx = local_rank
        if vis:
            ids = vis.split(',')
            if local_rank < len(ids) and ids[local_rank].isdigit():
                idx = int(ids[local_rank])
        h = pynvml.nvmlDeviceGetHandleByIndex(idx)
        bus = pynvml.nvmlDeviceGetPciInfo(h).busId
        if isinstance(bus, bytes):
            bus = bus.decode()
    except Exception:
        bus = None
    if not bus:
        return None
    bus = bus.lower()
    for cand in (bus, bus[-12:], '0000:' + bus[-7:]):       # nvml prints an 8-digit domain, sysfs a 4-digit one
        p = '/sys/bus/pci/devices/%s/numa_node' % cand
        if os.path.exists(p):
            try:
                n = int(open(p).read().strip())
                return n if n >= 0 else None
            except Exception:
                return None
    return None


def pin_rank(local_rank, local_world):
    """Pin this process to its share of the CPUs: the GPU's NUMA node (when known) intersected with the CPUs the process
    may use, split evenly among the ranks that land on the same node.  Returns a dict describing what was done."""
    try:
        allowed = sorted(os.sched_getaffinity(0))
    except AttributeError:
        return {'pinned': False, 'why': 'sched_getaffinity unavailable'}
    info = {'pinned': False, 'allowed': len(allowed)}
    node = gpu_numa_node(local_rank)
    cpus, peers, my_slot = allowed, local_world, local_rank
    if node is not None:
        try:
            node_cpus = set(_parse_cpulist(open('/sys/devices/system/node/node%d/cpulist' % node).read()))
            inter = [c for c in allowed if c in node_cpus]
            if inter:
                cpus = inter
                # ranks sharing this node: assume GPUs are spread evenly over the nodes in index order
                n_nodes = len([d for d in os.listdir('/sys/devices/system/node') if d.startswith('node') and d[4:].isdigit()])
                per_node = max(1, (local_world + n_nodes - 1) // n_nodes)
                peers = min(per_node, local_world)
                my_slot = local_rank % per_node
                info['numa_node'] = node
        except Exception:
            pass
    if peers > 1 and len(cpus) >= 2 * peers:
        share = len(cpus) // peers
        cpus = cpus[my_slot * share:(my_slot + 1) * share]
    try:
        os.sched_setaffinity(0, cpus)
        info.update(pinned=True, cpus=len(cpus), first=cpus[0], last=cpus[-1])
    except Exception as ex:
        info['why'] = str(ex)
    return info
