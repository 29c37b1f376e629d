"""Speculator training services (public names of reference ``speculator/train_speculator_utils.py``):
``generate``, ``stage1_loss``, ``stage2_loss``, ``do_ckpt``, ``train_speculator``, the ``Embed*`` base models
(forward returns hidden states next to the logits) and their registry
(``embedllama.{7b,8b}``, ``embedgpt_bigcode.20b``, ``embedmixtral.8x7b``)."""
from __future__ import annotations

import os
import time
from typing import Callable, Optional, Union

import torch
import torch.distributed as dist
import torch.nn as nn
import torch.nn.functional as F

from fms_fsdp_b200 import ops
from fms_fsdp_b200.models.llama import LLaMA, LLaMAConfig
from fms_fsdp_b200.parallel.tensor_parallel import refuse_unsupported_base, tp_all_gather_last, tp_all_reduce


# ---------------------------------------------------------------------------------- base models
def _only_causal_contiguous(mask, position_ids):
    """The Embed* forwards keep the reference's parameter list (``train_speculator_utils.py:432-441``); the frozen base model
    here always runs causal attention over contiguous positions (offset by the KV cache), which is all the trainer uses."""
    if mask is not None or position_ids is not None:
        raise NotImplementedError("explicit attention masks / position ids are not supported by the frozen base models")


class EmbedLLaMA(LLaMA):
    """Frozen LLaMA whose forward can also return the final hidden states ("embeds") and a KV cache.
    Inference only: prefill uses the engine's flash attention; single-token decode steps attend over the
    cache with SDPA.  With ``shard_llama_for_tp`` applied, row-parallel outputs are all-reduced.
    Reference: ``speculator/train_speculator_utils.py:464-492``."""

    def __init__(self, config: Optional[LLaMAConfig] = None, device=None, dtype=None, **kwargs):
        super().__init__(config, device, dtype, **kwargs)
        refuse_unsupported_base(self.config)

    def forward(self, x, mask=None, position_ids=None, past_key_value_states=None, use_cache=False,
                only_last_token=False, attn_algorithm=None, include_embeds=False):
        _only_causal_contiguous(mask, position_ids)
        tp = getattr(self, "_tp_group", None)
        B, S = x.shape
        h = self.shared(x)
        past = past_key_value_states
        pos0 = 0 if past is None else past[0][0].size(1)
        new_cache = []
        tab = self.rot_emb.table(h.device, pos0 + S)
        for li, blk in enumerate(self.layers):
            a = blk.attn
            qkv = a.in_proj.qkv_fused(blk.ln(h))
            K = ops.kernels_for(qkv)
            K.rope_(qkv.view(B * S, -1), tab, S, a.nheads, a.kvheads, a.head_dim, a.head_dim, False, pos0)
            if past is None and not use_cache:
                ctx = ops.attention(qkv, a.nheads, a.kvheads, a.head_dim)
            else:
                t = qkv.view(B, S, a.nheads + 2 * a.kvheads, a.head_dim)
                q, k, v = t[:, :, :a.nheads], t[:, :, a.nheads:a.nheads + a.kvheads], t[:, :, a.nheads + a.kvheads:]
                if past is not None:
                    k = torch.cat([past[li][0], k], dim=1)
                    v = torch.cat([past[li][1], v], dim=1)
                new_cache.append((k, v))
                ctx = F.scaled_dot_product_attention(
                    q.transpose(1, 2), k.transpose(1, 2), v.transpose(1, 2), is_causal=(past is None),
                    enable_gqa=(a.kvheads != a.nheads)).transpose(1, 2).reshape(B, S, a.nheads * a.head_dim)
            if tp is None:
                h = a.dense(ctx, residual=h)
                h = blk.ff_sub_layer.w2(ops.swiglu(blk.ff_sub_layer.wg1_fused(blk.ff_ln(h))), residual=h)
            else:
                h = h + tp_all_reduce(a.dense(ctx), tp)
                h = h + tp_all_reduce(blk.ff_sub_layer.w2(ops.swiglu(blk.ff_sub_layer.wg1_fused(blk.ff_ln(h)))), tp)
        embeds = self.dec_norm(h)
        if only_last_token:
            embeds = embeds[:, -1, :]
        logits = self.shared(embeds, reverse=True)
        if tp is not None:
            logits = tp_all_gather_last(logits, tp)
        out = [logits]
        if use_cache:
            out.append(new_cache)
        if include_embeds:
            out.append(embeds)
        return out[0] if len(out) == 1 else tuple(out)


class _GPTBigCodeBlock(nn.Module):
    def __init__(self, d, nheads, hidden, eps):
        super().__init__()
        self.nheads, self.hd = nheads, d // nheads   # nheads becomes the LOCAL head count under tensor parallelism
        self.tp_group = None
        self.ln = nn.LayerNorm(d, eps=eps)
        self.ff_ln = nn.LayerNorm(d, eps=eps)
        self.qkv = nn.Linear(d, d + 2 * self.hd)  # multi-query attention: one shared k/v head
        self.dense = nn.Linear(d, d)
        self.w1, self.w2 = nn.Linear(d, hidden), nn.Linear(hidden, d)

    def forward(self, h, past=None, use_cache=False):
        B, S, _ = h.shape
        Dq = self.nheads * self.hd
        q, k, v = self.qkv(self.ln(h)).split([Dq, self.hd, self.hd], dim=-1)
        if past is not None:
            k, v = torch.cat([past[0], k], 1), torch.cat([past[1], v], 1)
        ctx = F.scaled_dot_product_attention(q.view(B, S, self.nheads, self.hd).transpose(1, 2), k.unsqueeze(1),
                                             v.unsqueeze(1), is_causal=(past is None), enable_gqa=True)
        red = (lambda t: t) if self.tp_group is None else (lambda t: tp_all_reduce(t, self.tp_group))
        h = h + red(self.dense(ctx.transpose(1, 2).reshape(B, S, Dq)))
        h = h + red(self.w2(F.gelu(self.w1(self.ff_ln(h)), approximate="tanh")))
        return h, ((k, v) if use_cache else None)


class EmbedGPTBigCode(nn.Module):
    """GPT-BigCode (MQA, learned absolute positions, LayerNorm, GELU MLP) returning hidden states.
    Reference: ``speculator/train_speculator_utils.py:430-461``."""

    def __init__(self, vocab=49152, emb_dim=6144, nheads=48, nlayers=52, max_pos=8192, hidden_mult=4, eps=1e-5, **_):
        super().__init__()
        self.emb = nn.Embedding(vocab, emb_dim)
        self.pos = nn.Embedding(max_pos, emb_dim)
        self.layers = nn.ModuleList([_GPTBigCodeBlock(emb_dim, nheads, hidden_mult * emb_dim, eps) for _ in range(nlayers)])
        self.dec_norm = nn.LayerNorm(emb_dim, eps=eps)
        self.head = nn.Linear(emb_dim, vocab, bias=False)

    def reset_parameters(self):
        """GPT-2 style init (needed after ``to_empty`` when no checkpoint is given: the storage is uninitialised)."""
        for m in self.modules():
            if isinstance(m, (nn.Linear, nn.Embedding)):
                nn.init.normal_(m.weight, std=0.02)
                if getattr(m, "bias", None) is not None:
                    nn.init.zeros_(m.bias)
            elif isinstance(m, nn.LayerNorm):
                nn.init.ones_(m.weight)
                nn.init.zeros_(m.bias)

    def forward(self, x, mask=None, position_ids=None, past_key_value_states=None, use_cache=False,
                only_last_token=False, attn_algorithm=None, include_embeds=False):
        _only_causal_contiguous(mask, position_ids)
        past = past_key_value_states
        p0 = 0 if past is None else past[0][0].size(1)
        h = self.emb(x) + self.pos(torch.arange(p0, p0 + x.size(1), device=x.device))[None]
        cache = []
        for i, blk in enumerate(self.layers):
            h, c = blk(h, None if past is None else past[i], use_cache)
            cache.append(c)
        embeds = self.dec_norm(h)
        if only_last_token:
            embeds = embeds[:, -1, :]
        logits = self.head(embeds)
        if getattr(self, "_tp_group", None) is not None:
            logits = tp_all_gather_last(logits, self._tp_group)
        out = [logits] + ([cache] if use_cache else []) + ([embeds] if include_embeds else [])
        return out[0] if len(out) == 1 else tuple(out)


class _MoE(nn.Module):
    def __init__(self, d, hidden, n_experts, top_k):
        super().__init__()
        self.top_k = top_k
        self.gate = nn.Linear(d, n_experts, bias=False)
        self.w1 = nn.Parameter(torch.empty(n_experts, 2 * hidden, d))
        self.w2 = nn.Parameter(torch.empty(n_experts, d, hidden))
        self.reset_parameters()

    def reset_parameters(self):
        for w in (self.gate.weight, self.w1, self.w2):
            nn.init.trunc_normal_(w, std=0.02)

    def forward(self, x):
        B, S, D = x.shape
        xf = x.reshape(-1, D)
        w, idx = torch.topk(torch.softmax(self.gate(xf).float(), -1), self.top_k, dim=-1)
        w = (w / w.sum(-1, keepdim=True)).to(x.dtype)
        out = torch.zeros_like(xf)
        for e in range(self.w1.size(0)):
            tok, slot = torch.where(idx == e)
            if tok.numel() == 0:
                continue
            g, u = (xf[tok] @ self.w1[e].t()).chunk(2, dim=-1)
            out.index_add_(0, tok, (F.silu(g) * u) @ self.w2[e].t() * w[tok, slot].unsqueeze(-1))
        return out.view(B, S, D)


class EmbedMixtral(EmbedLLaMA):
    """Mixtral = the LLaMA block with a top-2-of-8 sparse MoE feed-forward; returns hidden states.
    Reference: ``speculator/train_speculator_utils.py:495-523``."""

    def __init__(self, config: Optional[LLaMAConfig] = None, n_experts=8, top_k=2, **kw):
        super().__init__(config, **kw)
        for blk in self.layers:
            blk.moe = _MoE(self.config.emb_dim, self.config.hidden_dim, n_experts, top_k)
            del blk.ff_sub_layer

    def reset_parameters(self):
        self.shared.reset_parameters()
        self.dec_norm.reset_parameters()
        for blk in self.layers:
            for m in (blk.ln, blk.ff_ln, blk.attn, blk.moe):
                m.reset_parameters()

    def forward(self, x, mask=None, position_ids=None, past_key_value_states=None, use_cache=False,
                only_last_token=False, attn_algorithm=None, include_embeds=False):
        _only_causal_contiguous(mask, position_ids)
        tp = getattr(self, "_tp_group", None)
        red = (lambda t: t) if tp is None else (lambda t: tp_all_reduce(t, tp))
        B, S = x.shape
        h = self.shared(x)
        past = past_key_value_states
        pos0 = 0 if past is None else past[0][0].size(1)
        tab = self.rot_emb.table(h.device, pos0 + S)
        cache = []
        for li, blk in enumerate(self.layers):
            a = blk.attn
            qkv = a.in_proj.qkv_fused(blk.ln(h))
            ops.kernels_for(qkv).rope_(qkv.view(B * S, -1), tab, S, a.nheads, a.kvheads, a.head_dim, a.head_dim, False, pos0)
            t = qkv.view(B, S, a.nheads + 2 * a.kvheads, a.head_dim)
            q, k, v = t[:, :, :a.nheads], t[:, :, a.nheads:a.nheads + a.kvheads], t[:, :, a.nheads + a.kvheads:]
            if past is not None:
                k, v = torch.cat([past[li][0], k], 1), torch.cat([past[li][1], v], 1)
            cache.append((k, v))
            ctx = F.scaled_dot_product_attention(q.transpose(1, 2), k.transpose(1, 2), v.transpose(1, 2),
                                                 is_causal=(past is None), enable_gqa=(a.kvheads != a.nheads))
            ctx = ctx.transpose(1, 2).reshape(B, S, -1)
            h = a.dense(ctx, residual=h) if tp is None else h + red(a.dense(ctx))
            h = h + red(blk.moe(blk.ff_ln(h)))
        embeds = self.dec_norm(h)
        if only_last_token:
            embeds = embeds[:, -1, :]
        logits = self.shared(embeds, reverse=True)
        if tp is not None:
            logits = tp_all_gather_last(logits, tp)
        out = [logits] + ([cache] if use_cache else []) + ([embeds] if include_embeds else [])
        return out[0] if len(out) == 1 else tuple(out)


_REGISTRY = {
    # 2-layer toys for CPU drills and tests (not reference variants)
    ("embedllama", "tiny"): lambda: EmbedLLaMA(LLaMAConfig(src_vocab_size=512, emb_dim=64, nheads=4, kvheads=2, nlayers=2,
                                                           multiple_of=16, max_expected_seq_len=256)),
    ("embedgpt_bigcode", "tiny"): lambda: EmbedGPTBigCode(vocab=512, emb_dim=64, nheads=4, nlayers=2, max_pos=256, hidden_mult=2),
    ("embedmixtral", "tiny"): lambda: EmbedMixtral(LLaMAConfig(src_vocab_size=512, emb_dim=64, nheads=4, kvheads=2, nlayers=2,
                                                               multiple_of=16, max_expected_seq_len=256), n_experts=4),
    ("embedllama", "7b"): lambda: EmbedLLaMA(LLaMAConfig(hidden_grow_factor=11008 / 4096, kvheads=32)),
    ("embedllama", "8b"): lambda: EmbedLLaMA(LLaMAConfig(src_vocab_size=128256, emb_dim=4096, nheads=32, kvheads=8,
                                                         nlayers=32, hidden_grow_factor=3.5, max_expected_seq_len=8192,
                                                         rope_theta=500000.0)),
    ("embedgpt_bigcode", "20b"): lambda: EmbedGPTBigCode(),
    ("embedmixtral", "8x7b"): lambda: EmbedMixtral(LLaMAConfig(emb_dim=4096, nheads=32, kvheads=8, nlayers=32,
                                                               hidden_grow_factor=14336 / 4096, max_expected_seq_len=32768,
                                                               rope_theta=1e6)),
}


def register_model(arch: str, variant: str, factory: Callable[[], nn.Module]):
    _REGISTRY[(arch, variant)] = factory


def get_model(arch: str, variant: str, model_path: Optional[str] = None, device_type="cuda", source="hf",
              distributed_strategy=None, group=None, dtype=torch.bfloat16):
    """Stand-in for ``fms.models.get_model``: build a registered base model and, when ``model_path`` holds an HF
    checkpoint (``source='hf'``), load its weights -- Llama, GPT-BigCode and Mixtral (reference adapters
    ``train_speculator_utils.py:526-569``); without a checkpoint the registered variant is built with random weights and
    that is said out loud.  ``distributed_strategy='tp'`` shards the base model (any of the three families) over ``group``."""
    dev = torch.device(device_type, torch.cuda.current_device()) if device_type == "cuda" else torch.device("cpu")
    has_ckpt = bool(model_path) and os.path.exists(os.path.join(model_path, "config.json"))
    if has_ckpt and arch in ("embedllama", "embedgpt_bigcode", "embedmixtral"):
        from fms_fsdp_b200.models import hf_loader
        if arch == "embedllama":
            model = hf_loader.load_hf_llama(model_path, "cpu", dtype, EmbedLLaMA)
        elif arch == "embedgpt_bigcode":
            model = hf_loader.load_hf_gpt_bigcode(model_path, EmbedGPTBigCode, "cpu", dtype)
        else:
            model = hf_loader.load_hf_mixtral(model_path, EmbedMixtral, "cpu", dtype)
    else:
        if int(os.environ.get("RANK", 0)) == 0:
            print(f"[get_model] no HF checkpoint at {model_path!r}: {arch}.{variant} is built with RANDOM weights")
        if (arch, variant) not in _REGISTRY:
            raise KeyError(f"unknown model {arch}.{variant}; registered: {sorted(_REGISTRY)}")
        with torch.device("meta"):
            model = _REGISTRY[(arch, variant)]()
        model.to_empty(device="cpu")
        if hasattr(model, "reset_parameters"):
            model.reset_parameters()
        model = model.to(dtype)
    if distributed_strategy == "tp" and group is not None and dist.get_world_size(group) > 1:
        from fms_fsdp_b200.parallel.tensor_parallel import shard_for_tp
        model = shard_for_tp(model, group)
    model = model.to(dev)
    for p in model.parameters():
        p.requires_grad_(False)
    return model


# ---------------------------------------------------------------------------------- generation
class _DecodeSession:
    """One autoregressive decode: owns the growing token matrix (pre-allocated once -- no O(n^2) re-concatenation), the
    KV cache handle and the per-step hidden states of the frozen base model."""

    def __init__(self, model, prompt: torch.Tensor, n_new: int, window: int, use_cache: bool, want_embeds: bool):
        self.model, self.window, self.use_cache, self.want_embeds = model, window, use_cache, want_embeds
        B, P = prompt.shape
        self.tokens = torch.empty(B, P + n_new, dtype=prompt.dtype, device=prompt.device)
        self.tokens[:, :P] = prompt
        self.filled = P
        self.cache = None
        self.hidden = []          # one [B, steps, D] block per model call

    def _model_input(self) -> torch.Tensor:
        if self.use_cache and self.cache is not None:
            return self.tokens[:, self.filled - 1: self.filled]          # only the newest token; the rest is cached
        return self.tokens[:, max(0, self.filled - self.window): self.filled]

    def next_logits(self) -> torch.Tensor:
        out = self.model(self._model_input(), past_key_value_states=self.cache, use_cache=self.use_cache,
                         include_embeds=self.want_embeds)
        if not (self.use_cache or self.want_embeds):
            return out[:, -1]
        if self.use_cache:
            self.cache = out[1]
        if self.want_embeds:
            self.hidden.append(out[-1])
        return out[0][:, -1]

    def append(self, next_tokens: torch.Tensor):
        self.tokens[:, self.filled] = next_tokens.reshape(-1)
        self.filled += 1


def _sample(logits: torch.Tensor, temperature: float, top_k: int) -> torch.Tensor:
    scores = logits.float() / temperature
    if top_k:
        kth = torch.topk(scores, top_k).values[:, -1:]
        scores = scores.masked_fill(scores < kth, float("-inf"))
    return torch.multinomial(torch.softmax(scores, dim=-1), 1)


def generate(model: Union[Callable, nn.Module], input_ids: torch.Tensor, max_seq_len: int = 2048,
             max_new_tokens: int = 256, temperature: float = 1.0, top_k: int = 10, do_sample: bool = True,
             num_beams: int = 1, use_cache: bool = False, contiguous_cache: bool = False, include_embeds: bool = True):
    """Decode ``max_new_tokens`` tokens after ``input_ids`` (greedy, or temperature / top-k sampling) and, with
    ``include_embeds``, also return the base model's final hidden state of every position it computed -- the
    training signal of stage 2 (same call contract as the reference's ``generate``, ``:28-118``)."""
    if num_beams != 1:
        raise NotImplementedError("beam search is not supported by generate()")
    if not torch.is_tensor(input_ids):
        raise RuntimeError("generate() needs the prompt as a tensor of token ids")
    single = input_ids.dim() == 1
    session = _DecodeSession(model, input_ids[None] if single else input_ids, max_new_tokens, max_seq_len,
                             use_cache, include_embeds)
    for _ in range(max_new_tokens):
        logits = session.next_logits()
        session.append(_sample(logits, temperature, top_k) if do_sample else logits.argmax(dim=-1))
    tokens = session.tokens[0] if single else session.tokens
    if not include_embeds:
        return tokens
    return tokens, (torch.cat(session.hidden, dim=-2) if session.hidden else None)


# -------------------------------------------------------------------------------------- losses
def _my_tp_slice(cfg, t, mesh):
    """Under TP every rank of the TP group ran the base model on the gathered batch; keep this rank's rows."""
    if cfg.sharding_strategy != "tp" or mesh is None:
        return t
    tp = mesh["tp"]
    return t.chunk(tp.size())[tp.get_local_rank()]


def _per_head_loss(preds: torch.Tensor, tokens: torch.Tensor, first_target: int, loss_fn, ddp_stats) -> torch.Tensor:
    """``preds`` [n_heads, B, N, V]; head i at position t is scored against ``tokens[:, first_target + i + t]``.  Adds
    each head's loss to ``ddp_stats[2 + i]`` and returns the sum over heads."""
    n_heads, _, width, vocab = preds.shape
    windows = tokens.unfold(1, width, 1)                      # [B, n_windows, width]; window j starts at token j
    total = preds.new_zeros((), dtype=torch.float32)
    for head in range(n_heads):
        target = windows[:, first_target + head]
        head_loss = loss_fn(preds[head].reshape(-1, vocab).float(), target.reshape(-1).long())
        ddp_stats[2 + head] += head_loss.detach()
        total = total + head_loss
    return total


def stage1_loss(cfg, model, speculator, base_model_input, input, loss_fn, ddp_stats, base_model_mesh):
    """Stage 1 (reference ``:122-171``): ONE parallel forward of the frozen base model over ground-truth text gives
    the hidden states; from the state at position t and the true tokens t+1.., head i predicts token t+2+i."""
    n = speculator.n_predict
    with torch.no_grad():
        _, hidden = model(base_model_input[:, : -(n + 1)], include_embeds=True, use_cache=False)
    hidden = _my_tp_slice(cfg, hidden, base_model_mesh).detach()
    preds = speculator(hidden, input[:, 1:])
    return _per_head_loss(preds, input, 2, loss_fn, ddp_stats), ddp_stats, input.numel()


def stage2_loss(cfg, model, speculator, base_model_input, input, loss_fn, ddp_stats, base_model_mesh):
    """Stage 2 (reference ``:175-242``): the batch is re-cut into many short prompts, the base model CONTINUES them
    (sampling, KV cache) and the speculator learns to predict the base model's own continuation."""
    n = speculator.n_predict
    with torch.no_grad():
        fan_out = cfg.stage2_batch_size // cfg.batch_size
        used = cfg.stage2_prompt_length * fan_out
        assert used <= cfg.seq_length, "Error: batch is too small for specified partition"
        prompts = base_model_input[:, :used].reshape(-1, cfg.stage2_prompt_length)
        text, hidden = generate(model, prompts, cfg.seq_length, cfg.stage2_seq_length, do_sample=True, use_cache=True,
                                include_embeds=True)
        text = _my_tp_slice(cfg, text, base_model_mesh)[:, -cfg.stage2_seq_length:]
        hidden = _my_tp_slice(cfg, hidden, base_model_mesh)[:, -cfg.stage2_seq_length: -n]
    preds = speculator(hidden.detach(), text[:, :-1].detach())
    return _per_head_loss(preds, text, 1, loss_fn, ddp_stats), ddp_stats, text.numel()


def do_ckpt(ckpt_save_path, reset=False):
    """Operator-triggered checkpoint: writing ``1`` into ``<ckpt_save_path>/do_ckpt`` asks the loop for a checkpoint at
    the next step; the loop acknowledges with ``reset=True``, which writes ``0`` back.
    Reference: ``speculator/train_speculator_utils.py:246-260``."""
    flag = os.path.join(ckpt_save_path, "do_ckpt")
    if not os.path.isfile(flag):
        return False
    if reset:
        with open(flag, "w") as fh:
            fh.write("0")
        return False
    with open(flag) as fh:
        return fh.read().strip() == "1"


# ---------------------------------------------------------------------------------------- loop
def train_speculator(cfg, model, speculator, local_rank, rank, train_loader, optimizer, scheduler, checkpointer,
                     start_step: int = 0, n_tok: int = 0, profiler=None, base_model_mesh=None):
    """Speculator training loop; ``speculator`` is a ``ShardedModel`` (NO_SHARD) around ``MLPSpeculator``.
    Reference: ``speculator/train_speculator_utils.py:263-427``."""
    model.eval()
    speculator.train()
    device = speculator.device
    is_cuda = device.type == "cuda"
    n_predict = speculator.module.n_predict
    ddp_stats = torch.zeros(2 + n_predict, device=device)
    start = loop_start = time.time()
    loss_fn = nn.CrossEntropyLoss()
    elapsed_tokens, step_tok = 0, 0
    world_size = int(os.environ.get("WORLD_SIZE", 1))
    for batch_idx, input in enumerate(train_loader, start=start_step + 1):
        if batch_idx > cfg.num_steps:
            break
        input = input.to(device)
        if cfg.sharding_strategy == "tp" and base_model_mesh is not None:
            tp = base_model_mesh["tp"]
            base_model_input = torch.zeros(tp.size() * input.size(0), input.size(1), dtype=input.dtype, device=device)
            dist.all_gather_into_tensor(base_model_input, input, group=tp.get_group())
        else:
            base_model_input = input
        optimizer.zero_grad()
        stage = stage1_loss if batch_idx <= cfg.stage2_start_step else stage2_loss
        holder = {}

        def closure(spec_module):
            loss, _, holder["tok"] = stage(cfg, model, spec_module, base_model_input, input, loss_fn, ddp_stats,
                                           base_model_mesh)
            return loss

        speculator.forward_backward_custom(closure)
        step_tok = holder["tok"]
        ddp_stats[0] += speculator.clip_grad_norm_(cfg.grad_clip_thresh)
        optimizer.step()
        scheduler.step()
        ddp_stats[1] += 1
        if profiler:
            profiler.step()

        if batch_idx % cfg.report_interval == 0:
            if world_size > 1:
                dist.all_reduce(ddp_stats, op=dist.ReduceOp.SUM)
            train_loss = ddp_stats[2:] / ddp_stats[1]
            g_norm = ddp_stats[0] / ddp_stats[1]
            elapsed_time = time.time() - loop_start
            elapsed_tokens += cfg.report_interval * world_size * step_tok
            if rank == 0:
                print(f"{time.time()}")
                print("step:", batch_idx)
                print("tokens seen:", n_tok + elapsed_tokens)
                for i in range(len(train_loss)):
                    print(f"loss {i + 1}:", train_loss[i].item())
                print("gradient norm:", g_norm.item())
                print(f"speed for these {cfg.report_interval} steps:", (time.time() - start) / cfg.report_interval)
                print("overall speed:", elapsed_time / (batch_idx - start_step))
                print("LR:", scheduler.get_last_lr())
                print("reserved memory:", torch.cuda.max_memory_reserved(device) if is_cuda else 0)
                print("active memory:", torch.cuda.max_memory_allocated(device) if is_cuda else 0)
                print("overall token per gpu per sec:", int(elapsed_tokens / world_size / elapsed_time))
                print("token per day:", int(elapsed_tokens / elapsed_time * 3600 * 24))
                print()
            start = time.time()
            ddp_stats.zero_()
        if is_cuda:
            torch.cuda.reset_peak_memory_stats(device)

        if batch_idx % cfg.checkpoint_interval == 0 or batch_idx == cfg.num_steps or do_ckpt(cfg.ckpt_save_path) is True:
            if is_cuda:
                torch.cuda.empty_cache()
            checkpointer.save(batch_idx, speculator, optimizer, train_loader if hasattr(train_loader, "dataset") else None,
                              tokens_seen=elapsed_tokens + n_tok)
            do_ckpt(cfg.ckpt_save_path, reset=True)
    return ddp_stats
