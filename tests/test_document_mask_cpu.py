"""Document-masked causal attention for packed rows (CPU tier): the segment table, the oracle ops against an independent
masked SDPA, per-document isolation of the model, the sharded engine against the single-process oracle, and the entry
points."""
import os
import re
import subprocess
import sys
import tempfile

import pytest
import torch
import torch.multiprocessing as mp
import torch.nn.functional as F

import test_engine_cpu as TE
from conftest import free_port
from fms_fsdp_b200 import ops
from fms_fsdp_b200.models.llama import LLaMA
from fms_fsdp_b200.ops import functional as FN
from fms_fsdp_b200.ops import torch_kernels as TK
from fms_fsdp_b200.utils.config_utils import get_model_config

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SEP = 7


def _table(rows):
    return ops.document_segments(torch.tensor(rows), SEP)


# ------------------------------------------------------------------------------------------- segment table
def test_document_segments_hand_written_rows():
    x = 3
    seg = _table([[x, x, x, x, x]])                     # no separator: one document
    assert seg.dtype == torch.int32 and seg.shape == (2, 5) and seg.is_contiguous()
    assert seg.tolist() == [[0, 0, 0, 0, 0], [4, 4, 4, 4, 4]]
    assert _table([[SEP, x, x, x]]).tolist() == [[0, 1, 1, 1], [0, 3, 3, 3]]          # separator at 0
    assert _table([[x, x, x, SEP]]).tolist() == [[0, 0, 0, 0], [3, 3, 3, 3]]          # separator at S-1
    assert _table([[x, SEP, SEP, x, x]]).tolist() == [[0, 0, 2, 3, 3], [1, 1, 2, 4, 4]]  # one-token document
    seg = _table([[x, SEP, x, x, x, x], [x, x, x, x, SEP, x]])       # rows are independent
    assert seg.tolist() == [[0, 0, 2, 2, 2, 2, 0, 0, 0, 0, 0, 5], [1, 1, 5, 5, 5, 5, 4, 4, 4, 4, 4, 5]]


def test_document_segments_invariants_on_random_rows():
    g = torch.Generator().manual_seed(0)
    tok = torch.randint(0, 12, (3, 200), generator=g)
    B, S = tok.shape
    seg = ops.document_segments(tok, SEP).long()
    s = torch.arange(S).repeat(B)
    assert bool((seg[0] <= s).all() and (s <= seg[1]).all())
    for r in range(2):
        assert bool((seg[r].view(B, S).diff(dim=1) >= 0).all())
    ends = seg[1][tok.reshape(-1) == SEP]
    assert torch.equal(ends, s[tok.reshape(-1) == SEP])    # a separator ends its own document


# ------------------------------------------------------------------------------------------- oracle ops
def _doc_ids(tokens):
    """document index of every position: separators before it in its row (independent of document_segments)"""
    is_sep = (tokens == SEP).long()
    return torch.cumsum(is_sep, dim=1) - is_sep


def _masked_sdpa(qkv, tokens, H, KVH, hd, scale):
    B, S, _ = qkv.shape
    t = qkv.float().view(B, S, H + 2 * KVH, hd)
    q, k, v = t[:, :, :H], t[:, :, H:H + KVH], t[:, :, H + KVH:]
    k = k.repeat_interleave(H // KVH, dim=2)
    v = v.repeat_interleave(H // KVH, dim=2)
    d = _doc_ids(tokens)
    pos = torch.arange(S)
    mask = (d.unsqueeze(2) == d.unsqueeze(1)) & (pos.view(1, S, 1) >= pos.view(1, 1, S))
    o = F.scaled_dot_product_attention(q.transpose(1, 2), k.transpose(1, 2), v.transpose(1, 2),
                                       attn_mask=mask.unsqueeze(1), scale=scale)
    return o.transpose(1, 2).reshape(B, S, H * hd)


def _packed_tokens(B, S, seed):
    g = torch.Generator().manual_seed(seed)
    tok = torch.randint(8, 50, (B, S), generator=g)
    tok[0, [5, 6, 17, S - 1]] = SEP          # consecutive separators (one-token document) and one at the end
    if B > 1:
        tok[1, [0, 30]] = SEP
    return tok


@pytest.mark.parametrize("H,KVH", [(4, 4), (4, 2)])
def test_attention_with_doc_matches_masked_sdpa(H, KVH):
    B, S, hd = 2, 40, 16
    torch.manual_seed(0)
    tok = _packed_tokens(B, S, 1)
    seg = ops.document_segments(tok, SEP)
    qkv = torch.randn(B, S, (H + 2 * KVH) * hd, requires_grad=True)
    do = torch.randn(B, S, H * hd)
    out = ops.attention(qkv, H, KVH, hd, doc=seg)
    (g,) = torch.autograd.grad(out, qkv, do)
    leaf = qkv.detach().requires_grad_(True)
    ref = _masked_sdpa(leaf, tok, H, KVH, hd, hd ** -0.5)
    (g_ref,) = torch.autograd.grad(ref, leaf, do)
    assert torch.allclose(out, ref, atol=1e-5, rtol=1e-4)
    assert torch.allclose(g, g_ref, atol=1e-5, rtol=1e-4)
    # the plain causal call is unchanged and differs from the masked one
    causal = ops.attention(qkv.detach(), H, KVH, hd)
    assert torch.allclose(causal, ops.attention(qkv.detach(), H, KVH, hd, doc=None))
    assert not torch.allclose(causal, out.detach(), atol=1e-3)


@pytest.mark.parametrize("precision", ["bf16", "fp8"])
def test_qkv_attention_with_doc_matches_masked_sdpa(precision):
    B, S, H, KVH, hd, D = 2, 40, 4, 2, 16, 64
    torch.manual_seed(0)
    tok = _packed_tokens(B, S, 2)
    seg = ops.document_segments(tok, SEP)
    dt = torch.float32 if precision == "bf16" else torch.bfloat16
    h = torch.randn(B, S, D).to(dt).requires_grad_(True)
    w = torch.nn.Parameter((0.2 * torch.randn((H + 2 * KVH) * hd, D)).to(dt))
    tab = TK.rope_table(S, hd)
    do = torch.randn(B, S, H * hd).to(dt)
    FN.set_gemm_precision(precision)
    try:
        out = ops.qkv_attention(h, w, tab, H, KVH, hd, doc=seg)
        gh, gw = torch.autograd.grad(out, (h, w), do)
        # independent: the same projection (fp8 forward on the fp8 path), RoPE, masked SDPA
        hl, wl = h.detach().requires_grad_(True), w.detach().requires_grad_(True)
        qkv = ops.linear(hl, wl) if precision == "fp8" else hl @ wl.t()
        qkv = TK.rope_(qkv.float().reshape(B * S, -1).clone(), tab, S, H, KVH, hd).view(B, S, -1) \
            if precision == "fp8" else qkv
    finally:
        FN.set_gemm_precision("bf16")
    if precision == "bf16":
        # differentiable RoPE for the reference gradients: rotate through the oracle op inside autograd
        qkv = ops.rope_(qkv.clone(), tab, S, H, KVH, hd)
        ref = _masked_sdpa(qkv, tok, H, KVH, hd, hd ** -0.5)
        rgh, rgw = torch.autograd.grad(ref, (hl, wl), do)
        assert torch.allclose(out, ref, atol=1e-5, rtol=1e-4)
        assert torch.allclose(gh, rgh, atol=1e-4, rtol=1e-3) and torch.allclose(gw, rgw, atol=1e-4, rtol=1e-3)
    else:
        ref = _masked_sdpa(qkv.detach(), tok, H, KVH, hd, hd ** -0.5)
        assert (out.float() - ref).abs().max() < 3e-2 * ref.abs().max()
        plain = ops.attention(qkv.detach().to(dt), H, KVH, hd)
        assert (out.float() - plain.float()).abs().max() > 5e-2 * ref.abs().max()   # the mask reached the kernel
        assert gh.isfinite().all() and gw.isfinite().all()


# ------------------------------------------------------------------------------------------- model isolation
def _tiny(doc):
    torch.manual_seed(0)
    cfg = get_model_config("llama2_tiny")
    cfg.doc_separator = SEP if doc else None
    m = LLaMA(cfg)
    m.reset_parameters()
    return m


def test_packed_documents_are_isolated_in_the_model():
    m = _tiny(doc=True)
    V = m.config.src_vocab_size
    g = torch.Generator().manual_seed(5)
    docs = [torch.randint(8, V, (n,), generator=g) for n in (13, 1, 20, 9)]
    docs = [torch.cat([d, torch.tensor([SEP])]) for d in docs[:-1]] + [docs[-1]]   # last one runs to the row end
    row = torch.cat(docs).unsqueeze(0)
    labels = torch.randint(0, V, row.shape, generator=g)

    def grads(x, y):
        m.zero_grad()
        logits = m(x)
        F.cross_entropy(logits.reshape(-1, V).float(), y.reshape(-1), reduction="sum").backward()
        return logits.detach(), {k: p.grad.clone() for k, p in m.named_parameters()}

    packed, g_packed = grads(row, labels)
    g_sum = {k: torch.zeros_like(v) for k, v in g_packed.items()}
    p0 = 0
    for d in docs:
        alone, g_doc = grads(d.unsqueeze(0), labels[:, p0:p0 + len(d)])
        assert torch.allclose(packed[:, p0:p0 + len(d)], alone, atol=1e-4, rtol=1e-4), p0
        for k in g_sum:
            g_sum[k] += g_doc[k]
        p0 += len(d)
    for k in g_sum:
        assert torch.allclose(g_packed[k], g_sum[k], atol=1e-4, rtol=1e-3), k
    # the same row without the mask attends across documents
    assert not torch.allclose(_tiny(doc=False)(row), packed, atol=1e-3)


def test_doc_separator_off_keeps_block_and_head_signatures():
    m = _tiny(doc=False)
    x = torch.randint(0, 100, (1, 16))
    h = m.engine_embed(x)
    assert isinstance(h, torch.Tensor)
    h2 = m.layers[0](h)
    assert isinstance(h2, torch.Tensor)
    assert torch.allclose(m.engine_head(h2, x), m.engine_head(h2, labels=x))   # labels still positional
    md = _tiny(doc=True)
    h, seg = md.engine_embed(x)
    assert seg.dtype == torch.int32 and not seg.requires_grad
    out = md.layers[0](h, seg)
    assert isinstance(out, tuple) and out[1] is seg
    assert torch.allclose(md.engine_head(out[0], seg, labels=x), md.engine_head(out[0], seg, x))


# ------------------------------------------------------------------------------------------- sharded engine
_plain_batch = TE._batch


def _doc_batch(rank, step):
    x = _plain_batch(rank, step)
    x[0, [0, 9, 10, TE.S - 1]] = SEP
    x[1, [3 + 5 * step + rank, 20]] = SEP
    return x


def _doc_config(variant):
    cfg = get_model_config(variant)
    cfg.doc_separator = SEP
    return cfg


def _patch_harness():
    TE._batch = _doc_batch
    TE.get_model_config = _doc_config


def _doc_worker(*args):
    _patch_harness()
    TE._worker(*args)


@pytest.mark.parametrize("ac", ["1", "1/2"])
def test_world2_fsdp_with_document_mask_matches_oracle(ac, monkeypatch):
    outdir = tempfile.mkdtemp()
    mp.spawn(_doc_worker, args=(2, free_port(), "fsdp", 0, ac, outdir, None), nprocs=2, join=True)
    out = torch.load(os.path.join(outdir, "out.pt"), weights_only=False)
    monkeypatch.setattr(TE, "_batch", _doc_batch)
    monkeypatch.setattr(TE, "get_model_config", _doc_config)
    TE._check(out, 2)
    # the oracle itself saw masked attention: a different trajectory than the plain model on the same batches
    monkeypatch.setattr(TE, "get_model_config", get_model_config)
    assert TE._oracle(2)[0] != pytest.approx(out["losses"], rel=1e-6, abs=1e-6)


# ------------------------------------------------------------------------------------------- entry points
def _train(data, ckpt, *extra):
    from test_real_data_entrypoint import _corpus
    if not os.path.isdir(data):
        _corpus(data)
    cmd = [sys.executable, os.path.join(ROOT, "main_training_llama.py"), "--model_variant=llama2_tiny",
           "--use_dummy_dataset=False", f"--data_path={data}", "--datasets=dataset_1,dataset_2", "--weights=2,1",
           "--file_type=arrow", "--col_name=tokens", "--logical_shards=8", "--num_workers=1", "--seq_length=32",
           "--vocab_size=512", "--batch_size=2", "--eos_token=0", "--num_steps=3", "--report_interval=1",
           "--checkpoint_interval=100", f"--ckpt_save_path={ckpt}", f"--ckpt_load_path={ckpt}",
           "--sharding_strategy=fsdp", "--comm_backend=gloo", "--use_torch_compile=False", *extra]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600, cwd=ROOT,
                       env=dict(os.environ, OMP_NUM_THREADS="1"))
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    return [float(x) for x in re.findall(r"^loss: ([0-9.eE+-]+)$", r.stdout, flags=re.M)]


def test_llama_entry_point_trains_with_the_document_mask(tmp_path):
    data = str(tmp_path / "data")
    masked = _train(data, str(tmp_path / "on"), "--document_attention_mask=True")
    plain = _train(data, str(tmp_path / "off"))
    assert len(masked) == 3 and all(l == l and l < 20 for l in masked), masked
    assert masked != plain, (masked, plain)


def test_mamba_entry_point_rejects_the_document_mask():
    import main_training_mamba
    with pytest.raises(ValueError, match="not supported for Mamba"):
        main_training_mamba.main(model_variant="mamba_tiny", document_attention_mask=True)
