"""Dependency stand-in for `ibm-fms` (not installable offline), used ONLY by `bench.py --impl reference`.

Plain PyTorch nn.Modules with the ibm-fms LLaMA architecture and attribute surface the unmodified
reference touches (fms.models.llama.{LLaMA, LLaMABlock, LLaMAConfig}; fms.modules.{attention,
embedding, feedforward, layernorm}).  No code of this repository's engine is imported here: GEMMs are
F.linear (cuBLAS), attention is F.scaled_dot_product_attention, everything else ATen/inductor --
i.e. exactly the kernel stack the reference runs (SURVEY.md section 2.5).
"""
