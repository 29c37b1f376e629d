"""Host-side logic of the fused all-gather queue (ops/cuda_kernels.py): a unit's prefetch request is spread over the GEMMs
that follow in proportion to their weight size, dependent requests are never split, leftovers are flushed as a plain
range gather.  The extension is loaded (it imports without a GPU) and its launch entry points are replaced by recorders."""
import pytest
import torch

try:
    from fms_fsdp_b200.ops import cuda_kernels as ck
except Exception as ex:   # extension not built in this checkout
    pytest.skip(f"fms_fsdp_b200._C not available: {ex!r}", allow_module_level=True)


class _Rec:
    def __init__(self):
        self.ag, self.plain = [], []

    def gemm_ag(self, a, b, out, layout, epi, residual, table, full, shard_bytes, begin, end, world, rank, flags, epoch, dep,
                **epi_args):
        self.ag.append((begin, end, bool(dep)))

    def p2p_gather_range(self, table, full, shard_bytes, begin, end):
        self.plain.append((begin, end))


def _meta(*shape):
    return torch.empty(*shape, dtype=torch.bfloat16, device="meta")


@pytest.fixture
def rec(monkeypatch):
    r = _Rec()
    monkeypatch.setattr(ck, "_C", r)
    monkeypatch.setattr(ck, "_AG_QUEUE", [])
    monkeypatch.setattr(ck, "AG_SPLIT", 1.0)
    return r


def _req(begin, end, dependent=False):
    return dict(table=None, full=None, shard_bytes=1, begin=begin, end=end, world=8, rank=0, flags=None, epoch=1,
                dependent=dependent)


def test_llama7b_block_forward_carries_exactly_one_unit(rec):
    T, D, QKV, F = 8192, 4096, 12288, 11008
    weights = [(QKV, D), (D, D), (2 * F, D), (D, F)]
    mb = 65536                                           # vectors (norm gains) occupy the first 64 KiB-aligned region
    total = mb + sum(n * k for n, k in weights) * 2
    req = _req(mb, total)
    ck.push_ag_request(req)
    x = {D: _meta(T, D), F: _meta(T, F)}
    for n, k in weights:                                 # the four forward GEMMs of a block
        assert ck._try_fused_gather(x[k], _meta(n, k), "nt", _meta(T, n), 0, None)
    assert req["consumed"] and not ck._AG_QUEUE
    spans = [(b, e) for b, e, _ in rec.ag]
    assert spans[0][0] == mb and spans[-1][1] == total
    assert all(a[1] == b[0] for a, b in zip(spans, spans[1:]))           # contiguous, no overlap
    assert [e - b for b, e in spans] == [n * k * 2 for n, k in weights]  # each GEMM carries its own weight size
    assert not rec.plain


def test_wgrad_uses_output_size_and_leftover_is_flushed(rec):
    req = _req(0, 10 * 65536)
    ck.push_ag_request(req)
    dy, x, dw = _meta(8192, 512), _meta(8192, 128), _meta(512, 128)       # tn: out is the weight-shaped operand
    assert ck._try_fused_gather(dy, x, "tn", dw, 0, None)
    assert rec.ag == [(0, 2 * 65536, False)] and not req["consumed"]     # 512*128*2 B = 2 chunks
    ck.flush_ag_request(req)
    assert rec.plain == [(2 * 65536, 10 * 65536)] and req["consumed"] and not ck._AG_QUEUE


def test_ineligible_gemm_leaves_prefetch_queued_but_flushes_dependent(rec):
    req = _req(0, 4 * 65536)
    ck.push_ag_request(req)
    small = _meta(64, 128)                                                 # M < 256: not a fused-epilogue GEMM
    assert not ck._try_fused_gather(small, _meta(256, 128), "nt", _meta(64, 256), 0, None)
    assert ck._AG_QUEUE == [req] and not rec.ag and not rec.plain


def test_split_factor_per_request(rec):
    req = _req(0, 64 * 65536)
    req["split"] = 0.5
    ck.push_ag_request(req)
    assert ck._try_fused_gather(_meta(8192, 256), _meta(1024, 256), "nt", _meta(8192, 1024), 0, None)
    assert rec.ag == [(0, 4 * 65536, False)]                               # half of 1024*256*2 B
