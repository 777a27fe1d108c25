"""CLIPTextModel with `inputs_embeds` — mirror of e4t/models/modeling_clip.py:9-82 (HF CLIP text tower naming:
text_model.embeddings.{token,position}_embedding, encoder.layers.{i}.{layer_norm1,self_attn.{q,k,v,out}_proj,
layer_norm2,mlp.fc1,mlp.fc2}, final_layer_norm; causal mask; quick_gelu).

Pre-training keeps the weights frozen, but dX must flow to the injected placeholder row (pretrain_e4t.py:630-634).  On
CUDA the tower runs on the e4t_b200 kernels (round 2, SURVEY.md §8 f-3): LayerNorm kernel, one fused q|k|v wgmma GEMM
with bias, the short-sequence causal attention kernel (77 tokens), out_proj / fc2 GEMMs with bias + residual epilogues,
quick-GELU kernel; every Function returns dX.  Domain tuning with --train_text_encoder (tuning_e4t.py:127-146) also
trains every text weight: each Function then returns its parameter gradients too (one dW GEMM for the fused q|k|v,
the deterministic embedding-gradient kernel for the token table, a column sum for the position table); a frozen
tower saves nothing for them and runs the same kernels as before.  CPU tensors (tokenizer-side utilities, tests of the module surface) take the plain
torch path below — it is not used by any GPU step."""
import json
import os
from dataclasses import dataclass
from typing import Optional

import torch
import torch.nn.functional as F
from torch import nn

from e4t._mixins import BaseOutput
from e4t_b200 import functional as FN
from e4t_b200 import ops


def _bf16(p):
    return FN.prepared(p, "bf16", lambda t: t.to(torch.bfloat16).contiguous())


def _f32(p):
    return p if p.dtype == torch.float32 else FN.prepared(p, "f32", lambda t: t.float().contiguous())


def _ln_k(norm, x):
    return FN.LayerNormFn.apply(x, _f32(norm.weight), _f32(norm.bias), norm.eps)


def _linear_k(lin, x, residual):
    """nn.Linear on the GEMM kernel; the fp32 master weight is passed for dW only when it is trained."""
    w = lin.weight
    return FN.LinearFn.apply(x, _bf16(w), _f32(lin.bias), residual, w if w.requires_grad else None)


@dataclass
class BaseModelOutputWithPooling(BaseOutput):
    last_hidden_state: torch.Tensor = None
    pooler_output: torch.Tensor = None


class CLIPTextConfig:
    def __init__(self, vocab_size=49408, hidden_size=768, intermediate_size=3072, num_hidden_layers=12,
                 num_attention_heads=12, max_position_embeddings=77, hidden_act="quick_gelu", layer_norm_eps=1e-5,
                 **kwargs):
        self.vocab_size = vocab_size
        self.hidden_size = hidden_size
        self.intermediate_size = intermediate_size
        self.num_hidden_layers = num_hidden_layers
        self.num_attention_heads = num_attention_heads
        self.max_position_embeddings = max_position_embeddings
        self.hidden_act = hidden_act
        self.layer_norm_eps = layer_norm_eps
        self.use_return_dict = True


class _Embeddings(nn.Module):
    def __init__(self, cfg):
        super().__init__()
        self.token_embedding = nn.Embedding(cfg.vocab_size, cfg.hidden_size)
        self.position_embedding = nn.Embedding(cfg.max_position_embeddings, cfg.hidden_size)

    def forward(self, input_ids=None, position_ids=None, inputs_embeds=None):
        if inputs_embeds is None:
            inputs_embeds = self.token_embedding(input_ids)
        n = inputs_embeds.shape[1]
        pos = self.position_embedding.weight[:n] if position_ids is None else self.position_embedding(position_ids)
        return inputs_embeds + pos

    def trained(self):
        return torch.is_grad_enabled() and (self.token_embedding.weight.requires_grad
                                            or self.position_embedding.weight.requires_grad)

    def forward_trained(self, input_ids=None, inputs_embeds=None):
        """Embedding sum on the device when a table is trained (--train_text_encoder), as bf16 activations: the token
        table takes its gradient from the embedding-gradient kernel, the position table from a column sum."""
        tok, pos = self.token_embedding.weight, self.position_embedding.weight
        if inputs_embeds is None:
            inputs_embeds = FN.TokenEmbeddingFn.apply(input_ids, tok) if tok.requires_grad else tok.detach()[input_ids]
        n = inputs_embeds.shape[1]
        if pos.requires_grad:
            return FN.PositionAddFn.apply(inputs_embeds.float(), pos[:n])
        return FN.as_bf16(inputs_embeds + pos[:n])


class _Attention(nn.Module):
    def __init__(self, cfg):
        super().__init__()
        d = cfg.hidden_size
        self.heads = cfg.num_attention_heads
        self.q_proj, self.k_proj, self.v_proj, self.out_proj = (nn.Linear(d, d) for _ in range(4))

    def _qkv(self):
        """q|k|v projection weights row-concatenated into one GEMM operand (cached bf16 copy) + fp32 bias."""
        ps = (self.q_proj, self.k_proj, self.v_proj)
        w = FN.prepared(self.q_proj.weight, ("qkv_bf16", self.k_proj.weight._version, self.v_proj.weight._version),
                        lambda t: torch.cat([p.weight.detach() for p in ps], dim=0).to(torch.bfloat16).contiguous())
        b = FN.prepared(self.q_proj.bias, ("qkv_bias", self.k_proj.bias._version, self.v_proj.bias._version),
                        lambda t: torch.cat([p.bias.detach() for p in ps], dim=0).float().contiguous())
        return w, b

    def forward_kernels(self, h, residual):
        D = h.shape[-1]
        w, b = self._qkv()
        ps = (self.q_proj, self.k_proj, self.v_proj)
        if torch.is_grad_enabled() and any(p.weight.requires_grad or p.bias.requires_grad for p in ps):
            qkv = FN.QKVLinearFn.apply(h, w, b, *(p.weight for p in ps), *(p.bias for p in ps))
        else:
            qkv = FN.LinearFn.apply(h, w, b, None, None)
        o = FN.SmallAttentionFn.apply(qkv, self.heads, (D // self.heads) ** -0.5, True)   # causal (modeling_clip.py:45-47)
        return _linear_k(self.out_proj, o, residual)

    def forward(self, x):
        B, N, D = x.shape
        h = self.heads
        q, k, v = (p(x).view(B, N, h, D // h).transpose(1, 2) for p in (self.q_proj, self.k_proj, self.v_proj))
        o = F.scaled_dot_product_attention(q, k, v, is_causal=True)              # causal mask (modeling_clip.py:45-47)
        return self.out_proj(o.transpose(1, 2).reshape(B, N, D))


class _MLP(nn.Module):
    def __init__(self, cfg):
        super().__init__()
        self.fc1 = nn.Linear(cfg.hidden_size, cfg.intermediate_size)
        self.fc2 = nn.Linear(cfg.intermediate_size, cfg.hidden_size)
        self.act = cfg.hidden_act

    def forward_kernels(self, h, residual):
        h = _linear_k(self.fc1, h, None)
        h = FN.ActFn.apply(h, ops.ACT_QUICK_GELU if self.act == "quick_gelu" else ops.ACT_GELU)
        return _linear_k(self.fc2, h, residual)

    def forward(self, x):
        h = self.fc1(x)
        h = h * torch.sigmoid(1.702 * h) if self.act == "quick_gelu" else F.gelu(h)
        return self.fc2(h)


class _Layer(nn.Module):
    def __init__(self, cfg):
        super().__init__()
        self.self_attn = _Attention(cfg)
        self.layer_norm1 = nn.LayerNorm(cfg.hidden_size, eps=cfg.layer_norm_eps)
        self.mlp = _MLP(cfg)
        self.layer_norm2 = nn.LayerNorm(cfg.hidden_size, eps=cfg.layer_norm_eps)

    def forward(self, x):
        if x.is_cuda:      # residual adds ride in the out_proj / fc2 GEMM epilogues
            x = self.self_attn.forward_kernels(_ln_k(self.layer_norm1, x), x)
            return self.mlp.forward_kernels(_ln_k(self.layer_norm2, x), x)
        x = x + self.self_attn(self.layer_norm1(x))
        return x + self.mlp(self.layer_norm2(x))


class _Encoder(nn.Module):
    def __init__(self, cfg):
        super().__init__()
        self.layers = nn.ModuleList([_Layer(cfg) for _ in range(cfg.num_hidden_layers)])

    def forward(self, x):
        for l in self.layers:
            x = l(x)
        return x


class _TextTransformer(nn.Module):
    def __init__(self, cfg):
        super().__init__()
        self.config = cfg
        self.embeddings = _Embeddings(cfg)
        self.encoder = _Encoder(cfg)
        self.final_layer_norm = nn.LayerNorm(cfg.hidden_size, eps=cfg.layer_norm_eps)


class CLIPTextModel(nn.Module):
    def __init__(self, config: Optional[CLIPTextConfig] = None, **kwargs):
        super().__init__()
        self.config = config if config is not None else CLIPTextConfig(**kwargs)
        self.text_model = _TextTransformer(self.config)

    @classmethod
    def from_pretrained(cls, path, subfolder=None, **kwargs):
        d = os.path.join(path, subfolder) if subfolder else path
        with open(os.path.join(d, "config.json")) as f:
            cfg = CLIPTextConfig(**json.load(f))
        m = cls(cfg)
        sd = {}
        for name in ("model.safetensors", "pytorch_model.bin"):
            f = os.path.join(d, name)
            if os.path.exists(f):
                if name.endswith(".safetensors"):
                    from safetensors.torch import load_file
                    sd = load_file(f, device="cpu")
                else:
                    sd = torch.load(f, map_location="cpu")
                break
        if not sd:
            raise FileNotFoundError(f"no text-encoder weights under {d} (model.safetensors / pytorch_model.bin)")
        missing, unexpected = m.load_state_dict(sd, strict=False)
        missing = [k for k in missing if "position_ids" not in k]
        unexpected = [k for k in unexpected if "position_ids" not in k]
        if missing or unexpected:
            raise RuntimeError(f"text encoder checkpoint mismatch: missing {missing[:5]} unexpected {unexpected[:5]}")
        return m

    @property
    def dtype(self):
        return self.text_model.final_layer_norm.weight.dtype

    @property
    def device(self):
        return self.text_model.final_layer_norm.weight.device

    def get_input_embeddings(self):
        return self.text_model.embeddings.token_embedding

    def resize_token_embeddings(self, new_num_tokens):
        old = self.text_model.embeddings.token_embedding
        if new_num_tokens == old.num_embeddings:
            return old
        new = nn.Embedding(new_num_tokens, old.embedding_dim).to(old.weight.device, old.weight.dtype)
        n = min(new_num_tokens, old.num_embeddings)
        with torch.no_grad():
            new.weight[:n] = old.weight[:n]
        new.weight.requires_grad_(old.weight.requires_grad)
        self.text_model.embeddings.token_embedding = new
        self.config.vocab_size = new_num_tokens
        return new

    def forward(self, input_ids=None, inputs_embeds=None, attention_mask=None, position_ids=None,
                output_attentions=None, output_hidden_states=None, return_dict=None):
        if input_ids is None and inputs_embeds is None:
            raise ValueError("You have to specify input_ids or inputs_embeds")
        if attention_mask is not None:
            raise NotImplementedError("attention_mask is never passed on the E4T path")
        if input_ids is not None:
            input_ids = input_ids.view(-1, input_ids.shape[-1])
        emb = self.text_model.embeddings
        src = emb.token_embedding.weight if inputs_embeds is None else inputs_embeds
        if src.is_cuda and position_ids is None and emb.trained():
            out_dtype = torch.promote_types(src.dtype, emb.position_embedding.weight.dtype)
            x = emb.forward_trained(input_ids=input_ids, inputs_embeds=inputs_embeds)
        else:
            x = emb(input_ids=input_ids, inputs_embeds=inputs_embeds, position_ids=position_ids)
            out_dtype = x.dtype
        if x.is_cuda:
            N, D = x.shape[1], x.shape[2]
            dh = D // self.config.num_attention_heads
            if N > 128 or dh > 64 or dh % 8 != 0:
                raise NotImplementedError(f"CLIP text tower on the e4t kernels needs N <= 128 and head dim <= 64 (got {N}, {dh})")
            x = _ln_k(self.text_model.final_layer_norm, self.text_model.encoder(FN.as_bf16(x))).to(out_dtype)
        else:
            x = self.text_model.final_layer_norm(self.text_model.encoder(x))
        pooled = x[:, 0]                                                         # modeling_clip.py:72
        if return_dict is False:
            return (x, pooled)
        return BaseModelOutputWithPooling(last_hidden_state=x, pooler_output=pooled)
