"""CPU: host-side helpers of bench.py that run before any GPU work."""
import os

import bench


def test_numa_binding_degrades_without_nvidia_smi():
    """No nvidia-smi / sysfs entry (this container): the rank stays unbound, says why, and its CPU affinity is untouched."""
    before = os.sched_getaffinity(0)
    info = bench.bind_to_gpu_numa_node(0)
    assert set(info) >= {"node", "cpus"}
    if info["node"] is None:
        assert os.sched_getaffinity(0) == before
    else:  # on a GPU box: bound to a non-empty subset
        assert 0 < info["cpus"] <= len(before) and os.sched_getaffinity(0) <= before
        os.sched_setaffinity(0, before)


def test_traffic_is_reported_only_for_a_capture_of_the_current_sources(tmp_path):
    """bench.py reports `roofline.traffic` only from a capture taken at the render kernels' current sources, and a
    committed profiles/traffic.json must be such a capture."""
    import json

    committed = os.path.join(bench.ROOT, "profiles", "traffic.json")
    if os.path.exists(committed):
        tj, _ = bench.traffic_capture(committed)
        assert tj is not None, "profiles/traffic.json belongs to other kernel sources: regenerate it (tools/make_traffic_json.py)"
        assert tj["dram_bytes_per_launch"] > 1e9 and set(tj["limiter"]) >= {"sample_issue_active_pct", "shade_issue_active_pct"}
    p = tmp_path / "traffic.json"
    assert bench.traffic_capture(str(p))[0] is None
    cap = {"kernel_sources_sha": bench.kernel_sources_sha(), "dram_bytes_per_launch": 2e9, "source": "these sources"}
    p.write_text(json.dumps(cap))
    assert bench.traffic_capture(str(p)) == (cap, "these sources")
    p.write_text(json.dumps(dict(cap, kernel_sources_sha="0" * 16)))
    assert bench.traffic_capture(str(p))[0] is None
