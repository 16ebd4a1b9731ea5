"""CPU tier of the host-resident slab: the load route's one-GPU rule, HostSlab's validation and chunking, and the ABI of the
staging entry points (declared, bound with matching arity, step-struct fields appended at the end)."""
import os
import re

import pytest
import torch

from helpers import ROOT


def test_load_route_host_slab_rule(tmp_path, monkeypatch):
    import coda_b200.datasets as ds
    path = str(tmp_path / "task.pt")
    torch.save(torch.rand(3, 40, 5), path)
    held = 3 * 40 * 5 * 4

    def host_slab_wanted(held_bytes, free_bytes, device_count, env):
        """Whether ``load_route`` loads the slab, scaled to ``held_bytes``, as one ``HostSlab``."""
        monkeypatch.setattr(ds, "_free_bytes", lambda index: free_bytes * held // held_bytes)
        monkeypatch.setattr(torch.cuda, "device_count", lambda: device_count)
        monkeypatch.setattr(torch.cuda, "current_device", lambda: 0)
        return ds.load_route(path, "cuda:0", env) == {"keep_dtype": False, "host": True}

    G = 1 << 30
    assert host_slab_wanted(100 * G, 80 * G, 1, {}) is True               # too large for the one GPU
    assert host_slab_wanted(10 * G, 80 * G, 1, {}) is False               # fits: the plain load
    assert host_slab_wanted(100 * G, 80 * G, 2, {}) is False              # several GPUs: per-GPU pieces instead
    assert host_slab_wanted(100 * G, 80 * G, 0, {}) is False
    assert host_slab_wanted(1, 80 * G, 4, {"CODA_B200_HOST_SLAB": "1"}) is True
    assert host_slab_wanted(100 * G, 80 * G, 1, {"CODA_B200_HOST_SLAB": "0"}) is False
    assert host_slab_wanted(100 * G, 80 * G, 1, {"CODA_B200_HOST_SLAB": ""}) is True


def test_shim_loads_host_slab_on_request(tmp_path, monkeypatch):
    import coda_b200.datasets as ds
    from coda.datasets import Dataset
    path = str(tmp_path / "task.pt")
    torch.save(torch.rand(3, 40, 5), path)
    calls = []
    monkeypatch.setattr(ds.Dataset, "__init__", lambda self, *a, **kw: calls.append((a, kw)))
    monkeypatch.setenv("CODA_B200_HOST_SLAB", "1")
    Dataset(path, "cuda:0")
    assert calls == [((path, "cuda:0"), {"keep_dtype": False, "host": True})]
    calls.clear()
    monkeypatch.setenv("CODA_B200_COMPACT_K", "2")                       # compaction keeps precedence
    Dataset(path, "cuda:0")
    assert calls[0][1].get("compact_k") == 2 and "host" not in calls[0][1]


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16, torch.bfloat16])
def test_host_slab_surface_and_chunks(dtype):
    from coda_b200 import HostSlab
    t = torch.rand(4, 1001, 6).to(dtype)
    s = HostSlab(t, "cuda:0", chunk_items=100)
    assert s.shape == (4, 1001, 6) and s.dtype == dtype and s.device == torch.device("cuda", 0)
    assert s.numel() == t.numel() and s.element_size() == t.element_size() and s.is_cuda
    assert s.chunk_items == 128                                           # whole 32-item scan tiles
    assert s.chunk_bytes() == 4 * 128 * 6 * t.element_size()
    assert HostSlab(t, "cuda:0", chunk_items=10 ** 9).chunk_items == 1024
    if dtype != torch.float32:
        assert HostSlab(t, "cuda:0", dtype=torch.float32).element_size() == 4
    with pytest.raises(TypeError):
        HostSlab(t, "cuda:0", dtype=torch.float16 if dtype == torch.bfloat16 else torch.bfloat16)
    with pytest.raises(ValueError):
        HostSlab(t.transpose(0, 1), "cuda:0")
    with pytest.raises(TypeError):
        HostSlab(t.double(), "cuda:0")
    with pytest.raises(TypeError):
        HostSlab(t, "cpu")


def test_host_stage_abi_is_declared_bound_and_appended():
    from coda_b200 import _native as nat
    from coda_b200 import build
    hdr = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "coda_b200.h")).read(), flags=re.S)
    for name, n in (("coda_b200_host_stage", 4), ("coda_b200_host_register", 2), ("coda_b200_host_unregister", 1)):
        m = re.search(r"\b" + name + r"\s*\(([^;]*?)\)\s*;", hdr, flags=re.S)
        assert m and m.group(1).count(",") + 1 == n == len(nat.SIGNATURES[name][1]), name
    assert "host_stage.cu" in build.SOURCES
    assert nat.VERSION == 203
    names = [f[0] for f in nat.StepStruct._fields_]
    assert names[-4:] == ["n_host", "host_shadow", "stage", "stage_off"]
    body = re.search(r"typedef struct coda_step \{(.*?)\} coda_step_t;", hdr, flags=re.S).group(1)
    assert re.findall(r"(\w+);", body)[-4:] == ["n_host", "host_shadow", "stage", "stage_off"]
