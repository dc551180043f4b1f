"""GPU: a context gives back all of its device memory when it is destroyed.  The device scratch of every operator family
(range tiers and the chunked host-pointer pipeline with its host timestamp scan, scalar(), topk, quantile, count_values,
subqueries, set operators) is owned by the context and freed with it, so creating, using and destroying contexts over
and over does not grow the process's device memory."""
import gc
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

T0, STEP = 1_700_000_000_000, 15_000
MiB = 1 << 20


def _words(rows, T):
    w = np.zeros((rows, (T + 31) // 32), np.uint32)
    for k in range(T):
        w[:, k // 32] |= np.uint32(1 << (k % 32))
    return w


def _process_memory():
    """() -> bytes of device memory NVML reports for this process on cuda:0; None when it reports none"""
    pynvml = pytest.importorskip("pynvml")
    import torch
    torch.zeros(1, device="cuda:0")  # this process's CUDA context, which the library's contexts share
    pynvml.nvmlInit()
    try:
        handle = pynvml.nvmlDeviceGetHandleByUUID("GPU-" + str(torch.cuda.get_device_properties(0).uuid))
    except Exception:
        handle = pynvml.nvmlDeviceGetHandleByIndex(0)

    def table():
        return {p.pid: int(p.usedGpuMemory) for p in pynvml.nvmlDeviceGetComputeRunningProcesses(handle)
                if p.usedGpuMemory is not None}
    pid = os.getpid()
    if pid not in table():
        # under a PID namespace NVML may list this process under another id: the one entry a probe allocation grows
        before = table()
        probe = torch.empty(256 * MiB, dtype=torch.uint8, device="cuda:0")
        grown = [q for q, b in table().items() if 256 * MiB <= b - before.get(q, 0) < 320 * MiB]
        del probe
        torch.cuda.empty_cache()
        if len(grown) != 1:
            return lambda: None
        pid = grown[0]
    return lambda: table().get(pid)


def _inputs():
    # chunked b2p_range_eval with an id column: more than 1.5 x 4 Mi rows of 8-row series (about 466 k series per
    # chunk), regular scrapes, so that every chunk is described by (offsets, t0, cadence) from the host scan
    S, N = 800_000, 8
    sid = np.repeat(np.arange(S, dtype=np.uint32), N)
    ts = T0 + np.tile(np.arange(N, dtype=np.int64) * STEP, S)
    val = np.tile(np.arange(N, dtype=np.float64), S)
    # grids of the operators above the range functions: one group of 1 000 rows (several chunks for topk and quantile)
    rng = np.random.default_rng(3)
    R, T = 1000, 40
    vals = rng.standard_normal((R, T))
    vals[rng.random((R, T)) < 0.3] = 1.0
    return dict(S=S, sid=sid, ts=ts, val=val, R=R, T=T, vals=vals, valid=_words(R, T))


def _cycle(x):
    from greptimedb_b200 import Context, make_params
    ctx = Context(0)
    try:
        p = make_params("rate", T0 + 60_000, T0 + 105_000, STEP, 60_000)
        out, valid, _ = ctx.range_eval(p, x["ts"], x["val"], sid=x["sid"])
        assert out.shape == (x["S"], 4) and (valid[:, 0] == 0xF).all()
        R, T, vals, words = x["R"], x["T"], x["vals"], x["valid"]
        one = np.zeros_like(words[:1])
        one[0] = words[0]
        s_out, s_valid = ctx.scalar_calculate(vals[:1], one, np.zeros(1, np.uint32))
        assert (s_out == vals[0]).all()
        gid = np.zeros(R, np.uint32)
        ctx.topk("topk", 3, vals, words, gid, 1, np.arange(R, dtype=np.uint32))
        ctx.group_quantile(0.9, vals, words, gid, 1)
        ctx.count_values(vals, words, gid, 1)
        q = make_params("sum_over_time", T0 + 300_000, T0 + (T - 1) * STEP, STEP, 300_000, filter_nan=False)
        ctx.subquery(q, T0, STEP, vals, words)
        key = (np.arange(R) % 7).astype(np.uint32)
        ctx.setop("or", vals, words, key, vals[:100], words[:100], key[:100], 7)
    finally:
        ctx.close()


def test_destroyed_contexts_give_back_their_device_memory():
    used = _process_memory()
    x = _inputs()
    _cycle(x)  # warm-up: the CUDA context, the library's modules and the runtime's own pools
    gc.collect()
    before = used()
    if before is None:
        pytest.skip("NVML does not report this process's device memory (e.g. under a PID namespace)")
    for _ in range(8):
        _cycle(x)
    gc.collect()
    after = used()
    print(f"device memory of this process: {before / MiB:.1f} MiB after the warm-up, {after / MiB:.1f} MiB after 8 cycles")
    assert after - before <= 4 * MiB, f"device memory grew by {(after - before) / MiB:.1f} MiB over 8 context lifetimes"
