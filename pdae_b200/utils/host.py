"""Host-side helpers."""
import os


def _cgroup_quota_cpus():
    """CPUs granted by the cgroup CPU quota (v2 `cpu.max`, v1 `cpu.cfs_quota_us` / `cpu.cfs_period_us`), or None."""
    try:
        quota, period = open("/sys/fs/cgroup/cpu.max").read().split()
        if quota != "max":
            return max(1, int(int(quota) / int(period)))
        return None
    except (OSError, ValueError):
        pass
    for d in ("/sys/fs/cgroup/cpu", "/sys/fs/cgroup/cpu,cpuacct", "/sys/fs/cgroup/cpuacct,cpu"):
        try:
            quota = int(open(os.path.join(d, "cpu.cfs_quota_us")).read())
            period = int(open(os.path.join(d, "cpu.cfs_period_us")).read())
        except (OSError, ValueError):
            continue
        return max(1, quota // period) if quota > 0 and period > 0 else None
    return None


def host_cores() -> int:
    """CPU cores this process may actually use: min(affinity, cgroup quota)."""
    n = len(os.sched_getaffinity(0)) if hasattr(os, "sched_getaffinity") else (os.cpu_count() or 1)
    q = _cgroup_quota_cpus()
    return max(1, min(n, q) if q else n)
