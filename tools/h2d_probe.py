"""Why does the pinned host->device rate differ between a plain `python bench.py` and torchrun on the same node
(VERDICT r1, Missing 1)?  Each variant runs in a fresh subprocess and prints its measured rate.
usage: python tools/h2d_probe.py            (runs all variants)
       python tools/h2d_probe.py VARIANT    (one variant, used by the parent)"""
import ctypes
import os
import subprocess
import sys
import time


def gpu_node_and_cpus(index=0):
    import torch
    p = torch.cuda.get_device_properties(index)
    path = "/sys/bus/pci/devices/%04x:%02x:%02x.0" % (p.pci_domain_id, p.pci_bus_id, p.pci_device_id)
    node = int(open(path + "/numa_node").read())
    cpus = open(path + "/local_cpulist").read().strip()
    ids = set()
    for part in cpus.split(","):
        if "-" in part:
            a, b = part.split("-"); ids.update(range(int(a), int(b) + 1))
        elif part:
            ids.add(int(part))
    return node, ids


def set_mempolicy_bind(node):
    libc = ctypes.CDLL(None, use_errno=True)
    mask = ctypes.c_ulong(1 << node)
    rc = libc.syscall(238, 2, ctypes.byref(mask), 64)  # set_mempolicy(MPOL_BIND, mask, maxnode)
    return rc, ctypes.get_errno()


def measure(src, dst, reps=5):
    import torch
    best = 0.0
    for _ in range(reps):
        a, z = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(); dst.copy_(src, non_blocking=True); z.record(); torch.cuda.synchronize()
        best = max(best, src.numel() / (a.elapsed_time(z) * 1e-3) / 1e9)
    return best


def run(variant):
    note = ""
    if variant == "affinity_before_import":
        # bind before torch / CUDA exist at all (node read from sysfs of the first NVIDIA device)
        import glob
        for d in sorted(glob.glob("/sys/bus/pci/devices/*")):
            try:
                if open(d + "/vendor").read().strip() == "0x10de" and open(d + "/class").read().startswith("0x0302"):
                    cpus = open(d + "/local_cpulist").read().strip()
                    ids = set()
                    for part in cpus.split(","):
                        if "-" in part:
                            a, b = part.split("-"); ids.update(range(int(a), int(b) + 1))
                        elif part:
                            ids.add(int(part))
                    os.sched_setaffinity(0, ids); note = "cpus " + cpus
                    break
            except Exception:
                pass
    import torch
    torch.cuda.set_device(0)
    node, ids = gpu_node_and_cpus(0)
    if variant in ("affinity", "affinity_mempolicy", "hostregister", "wc", "nccl_like_threads1"):
        os.sched_setaffinity(0, ids)
    if variant == "affinity_mempolicy":
        note = "set_mempolicy rc=%s" % (set_mempolicy_bind(node),)
    if variant == "nccl_like_threads1":
        torch.set_num_threads(1)
    n = 256 << 20
    dst = torch.empty(n, dtype=torch.uint8, device="cuda")
    if variant == "hostregister":
        buf = torch.empty(n, dtype=torch.uint8)
        buf.fill_(1)  # first touch on the bound CPUs
        rc = torch.cuda.cudart().cudaHostRegister(buf.data_ptr(), n, 0)
        note = "cudaHostRegister rc=%s" % (rc,)
        src = buf
    elif variant == "wc":
        import ctypes as C
        rt = C.CDLL("libcudart.so.12") if os.path.exists("/usr/local/cuda/lib64/libcudart.so.12") else None
        if rt is None:
            rt = C.CDLL("/usr/local/cuda/lib64/libcudart.so")
        p = C.c_void_p()
        rc = rt.cudaHostAlloc(C.byref(p), C.c_size_t(n), C.c_uint(4))  # cudaHostAllocWriteCombined
        note = "cudaHostAlloc(WC) rc=%d" % rc
        arr = (C.c_uint8 * n).from_address(p.value)
        src = torch.frombuffer(arr, dtype=torch.uint8)
    else:
        src = torch.empty(n, dtype=torch.uint8).pin_memory()
    t0 = time.time()
    g = measure(src, dst)
    # where did the pinned pages land?
    where = ""
    try:
        with open("/proc/self/numa_maps") as f:
            big = [ln for ln in f if "N0=" in ln or "N1=" in ln]
        tot = {}
        for ln in big:
            for tok in ln.split():
                if tok[:1] == "N" and "=" in tok and tok[1].isdigit():
                    k, v = tok.split("="); tot[k] = tot.get(k, 0) + int(v)
        where = " pages_by_node=%s" % tot
    except Exception:
        pass
    print("%-26s gpu_node=%d  H2D %.1f GB/s  %s%s" % (variant, node, g, note, where), flush=True)


if __name__ == "__main__":
    if len(sys.argv) > 1:
        run(sys.argv[1])
    else:
        for v in ("plain", "affinity", "affinity_before_import", "affinity_mempolicy", "hostregister", "wc", "nccl_like_threads1"):
            subprocess.run([sys.executable, __file__, v], timeout=120)
        # the same under torchrun (what the driver does for N > 1)
        subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "1", "--master-addr", "127.0.0.1",
                        "--master-port", "29533", __file__, "affinity"], timeout=180)
        env = dict(os.environ, OMP_NUM_THREADS="1")
        subprocess.run([sys.executable, __file__, "affinity"], env=env, timeout=120)
