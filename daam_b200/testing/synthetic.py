"""Synthetic, random-init stand-ins for the diffusers objects the hot path plugs into.

``diffusers`` is not installed on either box and there is no network, so the benchmark and the tests run
on plain-torch modules that expose exactly the surface the reference touches
(the reference's ``daam/trace.py:252-311``, ``daam/hook.py:95-127``):

* :class:`SyntheticAttention` -- the ``diffusers==0.21.2`` ``Attention`` module surface: ``to_q/to_k/to_v/to_out``,
  ``heads``, ``scale``, ``norm_cross``, ``upcast_attention``, ``upcast_softmax``, ``processor``/``set_processor`` and the
  helper methods the reference's hook calls (``prepare_attention_mask``, ``head_to_batch_dim``, ``batch_to_head_dim``,
  ``get_attention_scores``); SURVEY.md section 8c spells out the 0.21.2 semantics restated here.
* :class:`SyntheticUNet` -- a UNet2DConditionModel-shaped module tree (``down_blocks``/``mid_block``/``up_blocks`` whose
  class names contain ``CrossAttn``, ``.attentions[*].transformer_blocks[*].attn2``, ``config.sample_size``) in the
  SD-2.1-base and SDXL shapes. ``body='skeleton'`` keeps only the cross-attention layers (cheap; the operator-boundary
  benchmark and the CPU oracle use it), ``body='full'`` adds the resnets / self-attention / feed-forward so that
  "hooked vs un-hooked forward" is a meaningful overhead measurement.
* :class:`SyntheticPipeline` -- ``unet``, ``vae_scale_factor``, ``tokenizer.tokenize``, ``check_inputs``,
  ``image_processor.postprocess`` and a classifier-free-guidance loop that feeds the UNet ``[uncond, cond]`` batches.

These are fixtures: they contain no DAAM logic. The weights are random (default torch init), the data synthetic.
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from types import SimpleNamespace
from typing import List, Optional, Sequence

import torch
import torch.nn as nn
import torch.nn.functional as F

__all__ = [
    'SyntheticAttention', 'SDPAProcessor', 'SyntheticUNet', 'SyntheticPipeline', 'WhitespaceTokenizer',
    'UNetSpec', 'SD21_SPEC', 'SD21_768_SPEC', 'SDXL_SPEC', 'SD15_SPEC', 'TINY_SPEC', 'TINY15_SPEC', 'TINY96_SPEC', 'make_pipeline',
    'JointAttnProcessor', 'SyntheticJointAttention', 'JointTransformerBlock', 'SyntheticSD3Transformer',
    'SentencePieceTokenizer', 'SyntheticSD3Pipeline', 'SD3Spec', 'SD3_MEDIUM_SPEC', 'SD35_LARGE_SPEC', 'TINY_SD3_SPEC',
    'make_sd3_pipeline', 'flux_rotary_emb', 'FluxAttnProcessor', 'SyntheticFluxAttention', 'FluxTransformerBlock',
    'FluxSingleTransformerBlock', 'FluxPosEmbed', 'FluxSpec', 'FLUX_DEV_SPEC', 'FLUX_SCHNELL_SPEC', 'TINY_FLUX_SPEC',
    'SyntheticFluxTransformer', 'flux_image_ids', 'flux_pack', 'flux_unpack', 'SyntheticFluxPipeline',
    'make_flux_pipeline',
]


# ---------------------------------------------------------------------------------------------------------------
# Attention module with the diffusers 0.21.2 surface
# ---------------------------------------------------------------------------------------------------------------
class SDPAProcessor:
    """The un-hooked baseline: what diffusers' ``AttnProcessor2_0`` does (projections -> SDPA -> out projection)."""

    def __call__(self, attn, hidden_states, encoder_hidden_states=None, attention_mask=None):
        b, n, _ = hidden_states.shape
        ctx = hidden_states if encoder_hidden_states is None else encoder_hidden_states
        if encoder_hidden_states is not None and attn.norm_cross is not None:
            ctx = attn.norm_cross(ctx)
        h = attn.heads
        q = attn.to_q(hidden_states).view(b, n, h, -1).transpose(1, 2)
        k = attn.to_k(ctx).view(b, ctx.shape[1], h, -1).transpose(1, 2)
        v = attn.to_v(ctx).view(b, ctx.shape[1], h, -1).transpose(1, 2)
        out = F.scaled_dot_product_attention(q, k, v, attn_mask=attention_mask)
        out = out.transpose(1, 2).reshape(b, n, -1)
        return attn.to_out[1](attn.to_out[0](out))


class SyntheticAttention(nn.Module):
    """``diffusers.models.attention_processor.Attention`` (0.21.2) restated: same attributes, same helper semantics."""

    def __init__(self, query_dim: int, cross_attention_dim: Optional[int] = None, heads: int = 8, dim_head: int = 64,
                 upcast_attention: bool = False, upcast_softmax: bool = False):
        super().__init__()
        inner = heads * dim_head
        ctx_dim = query_dim if cross_attention_dim is None else cross_attention_dim
        self.heads = heads
        self.scale = dim_head ** -0.5
        self.upcast_attention = upcast_attention
        self.upcast_softmax = upcast_softmax
        self.norm_cross = None
        self.to_q = nn.Linear(query_dim, inner, bias=False)
        self.to_k = nn.Linear(ctx_dim, inner, bias=False)
        self.to_v = nn.Linear(ctx_dim, inner, bias=False)
        self.to_out = nn.ModuleList([nn.Linear(inner, query_dim), nn.Dropout(0.0)])
        self.processor = SDPAProcessor()

    def set_processor(self, processor):
        self.processor = processor

    def forward(self, hidden_states, encoder_hidden_states=None, attention_mask=None):
        return self.processor(self, hidden_states, encoder_hidden_states=encoder_hidden_states,
                              attention_mask=attention_mask)

    # -- helpers the reference hook calls (trace.py:261, 272-276, 297) --------------------------------------
    def prepare_attention_mask(self, attention_mask, target_length, batch_size):
        if attention_mask is None:
            return None
        if attention_mask.shape[-1] != target_length:
            attention_mask = F.pad(attention_mask, (0, target_length), value=0.0)
        if attention_mask.shape[0] < batch_size * self.heads:
            attention_mask = attention_mask.repeat_interleave(self.heads, dim=0)
        return attention_mask

    def head_to_batch_dim(self, tensor):
        b, n, c = tensor.shape
        h = self.heads
        return tensor.reshape(b, n, h, c // h).permute(0, 2, 1, 3).reshape(b * h, n, c // h)

    def batch_to_head_dim(self, tensor):
        bh, n, d = tensor.shape
        h = self.heads
        return tensor.reshape(bh // h, h, n, d).permute(0, 2, 1, 3).reshape(bh // h, n, d * h)

    def get_attention_scores(self, query, key, attention_mask=None):
        dtype = query.dtype
        if self.upcast_attention:
            query, key = query.float(), key.float()
        if attention_mask is None:
            base = torch.empty(query.shape[0], query.shape[1], key.shape[1], dtype=query.dtype, device=query.device)
            beta = 0
        else:
            base, beta = attention_mask, 1
        scores = torch.baddbmm(base, query, key.transpose(-1, -2), beta=beta, alpha=self.scale)
        del base
        if self.upcast_softmax:
            scores = scores.float()
        probs = scores.softmax(dim=-1)
        del scores
        return probs.to(dtype)


# ---------------------------------------------------------------------------------------------------------------
# UNet pieces
# ---------------------------------------------------------------------------------------------------------------
class _GEGLUFeedForward(nn.Module):
    def __init__(self, dim):
        super().__init__()
        self.proj = nn.Linear(dim, dim * 8)
        self.out = nn.Linear(dim * 4, dim)

    def forward(self, x):
        a, g = self.proj(x).chunk(2, dim=-1)
        return self.out(a * F.gelu(g))


class BasicTransformerBlock(nn.Module):
    def __init__(self, dim, heads, dim_head, ctx_dim, full: bool, upcast_attention: bool = False):
        super().__init__()
        self.full = full
        if full:
            self.norm1 = nn.LayerNorm(dim)
            self.attn1 = SyntheticAttention(dim, None, heads, dim_head, upcast_attention=upcast_attention)
            self.norm3 = nn.LayerNorm(dim)
            self.ff = _GEGLUFeedForward(dim)
        self.norm2 = nn.LayerNorm(dim)
        self.attn2 = SyntheticAttention(dim, ctx_dim, heads, dim_head, upcast_attention=upcast_attention)

    def forward(self, x, ctx):
        if self.full:
            x = x + self.attn1(self.norm1(x))
        x = x + self.attn2(self.norm2(x), encoder_hidden_states=ctx)
        if self.full:
            x = x + self.ff(self.norm3(x))
        return x


class Transformer2DModel(nn.Module):
    def __init__(self, channels, heads, dim_head, ctx_dim, depth, full, upcast_attention=False):
        super().__init__()
        self.norm = nn.GroupNorm(32 if channels % 32 == 0 else 1, channels, eps=1e-6)
        self.proj_in = nn.Linear(channels, channels)
        self.transformer_blocks = nn.ModuleList(
            [BasicTransformerBlock(channels, heads, dim_head, ctx_dim, full, upcast_attention) for _ in range(depth)])
        self.proj_out = nn.Linear(channels, channels)

    def forward(self, x, ctx):
        b, c, h, w = x.shape
        res = x
        y = self.norm(x).permute(0, 2, 3, 1).reshape(b, h * w, c)
        y = self.proj_in(y)
        for blk in self.transformer_blocks:
            y = blk(y, ctx)
        y = self.proj_out(y).reshape(b, h, w, c).permute(0, 3, 1, 2)
        return y + res


class ResnetBlock2D(nn.Module):
    def __init__(self, cin, cout, temb_dim, full):
        super().__init__()
        self.full = full
        if full:
            self.norm1 = nn.GroupNorm(32 if cin % 32 == 0 else 1, cin, eps=1e-5)
            self.conv1 = nn.Conv2d(cin, cout, 3, padding=1)
            self.time_emb_proj = nn.Linear(temb_dim, cout)
            self.norm2 = nn.GroupNorm(32 if cout % 32 == 0 else 1, cout, eps=1e-5)
            self.conv2 = nn.Conv2d(cout, cout, 3, padding=1)
        self.shortcut = nn.Conv2d(cin, cout, 1) if (cin != cout or not full) else None

    def forward(self, x, temb):
        if not self.full:
            return self.shortcut(x)
        h = self.conv1(F.silu(self.norm1(x)))
        h = h + self.time_emb_proj(F.silu(temb))[:, :, None, None]
        h = self.conv2(F.silu(self.norm2(h)))
        return h + (x if self.shortcut is None else self.shortcut(x))


class _Down(nn.Module):
    def __init__(self, c, full):
        super().__init__()
        self.conv = nn.Conv2d(c, c, 3, stride=2, padding=1) if full else None

    def forward(self, x):
        # ceil-sized like diffusers' stride-2 convolution (which the full body's conv is): odd sides round up
        return self.conv(x) if self.conv is not None else F.avg_pool2d(x, 2, ceil_mode=True)


class _Up(nn.Module):
    def __init__(self, c, full):
        super().__init__()
        self.conv = nn.Conv2d(c, c, 3, padding=1) if full else None

    def forward(self, x, size=None):
        # to the next skip's size (diffusers' upsample_size), which is twice the input unless a side was odd
        if size is None or tuple(size) == (2 * x.shape[-2], 2 * x.shape[-1]):
            x = F.interpolate(x, scale_factor=2.0, mode='nearest')
        else:
            x = F.interpolate(x, size=size, mode='nearest')
        return self.conv(x) if self.conv is not None else x


class _DownBlockBase(nn.Module):
    def __init__(self, cin, cout, temb_dim, n_layers, add_down, full, attn=None):
        super().__init__()
        self.resnets = nn.ModuleList([ResnetBlock2D(cin if i == 0 else cout, cout, temb_dim, full)
                                      for i in range(n_layers)])
        if attn is not None:
            self.attentions = nn.ModuleList([Transformer2DModel(cout, full=full, **attn) for _ in range(n_layers)])
        self.downsamplers = nn.ModuleList([_Down(cout, full)]) if add_down else None

    def forward(self, x, temb, ctx):
        skips = []
        for i, res in enumerate(self.resnets):
            x = res(x, temb)
            if hasattr(self, 'attentions'):
                x = self.attentions[i](x, ctx)
            skips.append(x)
        if self.downsamplers is not None:
            x = self.downsamplers[0](x)
            skips.append(x)
        return x, skips


class DownBlock2D(_DownBlockBase):
    pass


class CrossAttnDownBlock2D(_DownBlockBase):
    pass


class _UpBlockBase(nn.Module):
    def __init__(self, cin_prev, cout, skip_channels: Sequence[int], temb_dim, add_up, full, attn=None):
        super().__init__()
        res = []
        for i, sc in enumerate(skip_channels):
            res.append(ResnetBlock2D((cin_prev if i == 0 else cout) + sc, cout, temb_dim, full))
        self.resnets = nn.ModuleList(res)
        if attn is not None:
            self.attentions = nn.ModuleList(
                [Transformer2DModel(cout, full=full, **attn) for _ in range(len(skip_channels))])
        self.upsamplers = nn.ModuleList([_Up(cout, full)]) if add_up else None

    def forward(self, x, skips, temb, ctx):
        for i, res in enumerate(self.resnets):
            x = res(torch.cat([x, skips.pop()], dim=1), temb)
            if hasattr(self, 'attentions'):
                x = self.attentions[i](x, ctx)
        if self.upsamplers is not None:
            x = self.upsamplers[0](x, tuple(skips[-1].shape[-2:]) if skips else None)
        return x


class UpBlock2D(_UpBlockBase):
    pass


class CrossAttnUpBlock2D(_UpBlockBase):
    pass


class UNetMidBlock2DCrossAttn(nn.Module):
    def __init__(self, c, temb_dim, full, attn):
        super().__init__()
        self.resnets = nn.ModuleList([ResnetBlock2D(c, c, temb_dim, full), ResnetBlock2D(c, c, temb_dim, full)])
        self.attentions = nn.ModuleList([Transformer2DModel(c, full=full, **attn)])

    def forward(self, x, temb, ctx):
        x = self.resnets[0](x, temb)
        x = self.attentions[0](x, ctx)
        return self.resnets[1](x, temb)


@dataclass
class UNetSpec:
    """Shape of a UNet2DConditionModel. ``heads[i]``/``depth[i]`` belong to ``block_out_channels[i]``; ``depth`` 0
    means a block without cross-attention (``DownBlock2D``/``UpBlock2D``)."""
    name: str
    sample_size: int
    block_out_channels: Sequence[int]
    heads: Sequence[int]
    depth: Sequence[int]
    cross_attention_dim: int
    dim_head: Optional[int] = 64              # None: SD-1.x style, head_dim = channels // heads
    layers_per_block: int = 2
    mid_depth: Optional[int] = None          # transformer depth of the mid block (None: same as last block, min 1)
    in_channels: int = 4
    upcast_attention: bool = False
    tokens: int = 77


# public unet/config.json values of stabilityai/stable-diffusion-2-1-base and stabilityai/stable-diffusion-xl-base-1.0
SD21_SPEC = UNetSpec('sd21-base', 64, (320, 640, 1280, 1280), (5, 10, 20, 20), (1, 1, 1, 0), 1024)
# stabilityai/stable-diffusion-2-1 (the 768-pixel v-prediction model): same UNet, 96x96 latent -> latent_hw 9216
SD21_768_SPEC = UNetSpec('sd21-768', 96, (320, 640, 1280, 1280), (5, 10, 20, 20), (1, 1, 1, 0), 1024)
SDXL_SPEC = UNetSpec('sdxl-base', 128, (320, 640, 1280), (5, 10, 20), (0, 2, 10), 2048, mid_depth=10)
# runwayml/stable-diffusion-v1-5: 8 heads at every level, head dims 40 / 80 / 160
SD15_SPEC = UNetSpec('sd15', 64, (320, 640, 1280, 1280), (8, 8, 8, 8), (1, 1, 1, 0), 768, dim_head=None)
# a small tree with the SD-2.1 topology (15 located layers, factors 1/2/4, mid layer at factor 8) for CPU tests
TINY_SPEC = UNetSpec('tiny', 64, (64, 128, 128, 128), (1, 2, 2, 2), (1, 1, 1, 0), 96)
# the same topology with SD-1.x style head dims (40 / 80 / 80)
TINY15_SPEC = UNetSpec('tiny15', 64, (80, 160, 160, 160), (2, 2, 2, 2), (1, 1, 1, 0), 96, dim_head=None)
# the 768-pixel models' geometry (96x96 latent -> latent_hw 9216, daam/trace.py:32-33): layers at 96^2 / 48^2 / 24^2
# (9216 / 2304 / 576 query positions: partial 128-pixel tiles), mid layer at 12^2 (factor 8, skipped)
TINY96_SPEC = UNetSpec('tiny96', 96, (64, 128, 128, 128), (1, 2, 2, 2), (1, 1, 1, 0), 96)


class SyntheticUNet(nn.Module):
    """UNet2DConditionModel-shaped random-init network (see module docstring). ``forward(sample, t, ctx)``."""

    def __init__(self, spec: UNetSpec, body: str = 'skeleton'):
        super().__init__()
        assert body in ('skeleton', 'full')
        full = body == 'full'
        self.spec = spec
        self.config = SimpleNamespace(sample_size=spec.sample_size, in_channels=spec.in_channels,
                                      cross_attention_dim=spec.cross_attention_dim)
        ch = list(spec.block_out_channels)
        temb_dim = ch[0] * 4
        self.temb_dim = temb_dim
        self.time_embedding = nn.Sequential(nn.Linear(ch[0], temb_dim), nn.SiLU(), nn.Linear(temb_dim, temb_dim))
        self.conv_in = nn.Conv2d(spec.in_channels, ch[0], 3, padding=1)

        def attn_cfg(i):
            if spec.depth[i] == 0:
                return None
            return dict(heads=spec.heads[i], dim_head=spec.dim_head or ch[i] // spec.heads[i],
                        ctx_dim=spec.cross_attention_dim, depth=spec.depth[i], upcast_attention=spec.upcast_attention)

        downs, skip_ch = [], [ch[0]]
        cin = ch[0]
        for i, cout in enumerate(ch):
            last = i == len(ch) - 1
            cls = CrossAttnDownBlock2D if spec.depth[i] else DownBlock2D
            downs.append(cls(cin, cout, temb_dim, spec.layers_per_block, not last, full, attn_cfg(i)))
            skip_ch += [cout] * spec.layers_per_block + ([] if last else [cout])
            cin = cout
        self.down_blocks = nn.ModuleList(downs)

        mid_depth = spec.mid_depth if spec.mid_depth is not None else max(1, spec.depth[-1])
        self.mid_block = UNetMidBlock2DCrossAttn(ch[-1], temb_dim, full, dict(
            heads=spec.heads[-1], dim_head=spec.dim_head or ch[-1] // spec.heads[-1],
            ctx_dim=spec.cross_attention_dim, depth=mid_depth,
            upcast_attention=spec.upcast_attention))

        ups = []
        cin = ch[-1]
        for j, i in enumerate(reversed(range(len(ch)))):
            cout = ch[i]
            last = j == len(ch) - 1
            sk = [skip_ch.pop() for _ in range(spec.layers_per_block + 1)]
            cls = CrossAttnUpBlock2D if spec.depth[i] else UpBlock2D
            ups.append(cls(cin, cout, sk, temb_dim, not last, full, attn_cfg(i)))
            cin = cout
        self.up_blocks = nn.ModuleList(ups)
        self.conv_norm_out = nn.GroupNorm(32 if ch[0] % 32 == 0 else 1, ch[0])
        self.conv_out = nn.Conv2d(ch[0], spec.in_channels, 3, padding=1)

    def _time_embed(self, t, batch, dtype, device):
        half = self.spec.block_out_channels[0] // 2
        freqs = torch.exp(-math.log(10000.0) * torch.arange(half, device=device, dtype=torch.float32) / half)
        arg = torch.as_tensor(t, device=device, dtype=torch.float32).reshape(-1, 1).expand(batch, 1) * freqs[None]
        emb = torch.cat([arg.sin(), arg.cos()], dim=-1).to(dtype)
        return self.time_embedding(emb)

    def forward(self, sample, timestep, encoder_hidden_states):
        temb = self._time_embed(timestep, sample.shape[0], sample.dtype, sample.device)
        x = self.conv_in(sample)
        skips = [x]
        for blk in self.down_blocks:
            x, s = blk(x, temb, encoder_hidden_states)
            skips += s
        x = self.mid_block(x, temb, encoder_hidden_states)
        for blk in self.up_blocks:
            x = blk(x, skips, temb, encoder_hidden_states)
        return self.conv_out(F.silu(self.conv_norm_out(x)))


# ---------------------------------------------------------------------------------------------------------------
# Pipeline
# ---------------------------------------------------------------------------------------------------------------
class WhitespaceTokenizer:
    """CLIP-tokenizer stand-in: lower-cased whitespace pieces carrying the ``</w>`` end-of-word marker."""

    def tokenize(self, text: str) -> List[str]:
        return [w + '</w>' for w in text.lower().split()]


class _ImageProcessor:
    def postprocess(self, image, output_type='pil'):
        return [image[i] for i in range(image.shape[0])]


class SyntheticPipeline:
    """A StableDiffusionPipeline-shaped driver around :class:`SyntheticUNet`.

    Per denoising step it copies the step's inputs (latents, text embeddings, timestep; kept in pinned host memory when
    the UNet lives on a GPU) to the device, runs the UNet on the CFG batch ``[uncond x N, cond x N]`` and reads the
    guided noise estimate's mean back to the host -- the host<->device traffic ``bench.py`` counts for its ``e2e`` figure.

    ``cuda_graph=True`` replays the step's device work (UNet forward + guidance update) from a CUDA graph: the first step
    of a configuration runs eagerly, the second is captured, later steps and later calls replay it. Attention processors
    installed at capture time (e.g. a tracer's) are part of the graph; the graph is re-captured when they change.
    """

    def __init__(self, unet: SyntheticUNet, dtype=torch.float32, device='cpu', seed: int = 0,
                 cuda_graph: bool = False):
        self.unet = unet.to(device=device, dtype=dtype).eval()
        self.dtype, self.device = dtype, torch.device(device)
        self.vae_scale_factor = 8
        self.tokenizer = WhitespaceTokenizer()
        self.image_processor = _ImageProcessor()
        self.seed = seed
        self.cuda_graph = cuda_graph and self.device.type == 'cuda'
        self.h2d_bytes_per_step = 0
        self.d2h_bytes_per_step = 0
        self._graphs = {}
        self._attn = [m for m in self.unet.modules() if isinstance(m, SyntheticAttention)]

    def check_inputs(self, prompt, height=None, width=None, callback_steps=None, negative_prompt=None,
                     prompt_embeds=None, negative_prompt_embeds=None, *args, **kwargs):
        """diffusers' SD ``check_inputs`` parameter order, so that callers bind ``negative_prompt`` and
        ``prompt_embeds`` as they do there."""
        if prompt is None and prompt_embeds is None:
            raise ValueError('Provide either `prompt` or `prompt_embeds`')
        if prompt is not None and prompt_embeds is not None:
            raise ValueError('Cannot forward both `prompt` and `prompt_embeds`')
        if prompt is not None and not isinstance(prompt, (str, list)):
            raise ValueError('`prompt` has to be of type `str` or `list`')
        if negative_prompt is not None and not isinstance(negative_prompt, (str, list)):
            raise ValueError('`negative_prompt` has to be of type `str` or `list`')

    def encode(self, prompts: List[str], generator: torch.Generator):
        """Synthetic text encoder: seeded gaussian embeddings, [uncond x N, cond x N] like diffusers' CFG concat."""
        n, spec = len(prompts), self.unet.spec
        emb = torch.randn(2 * n, spec.tokens, spec.cross_attention_dim, generator=generator, dtype=torch.float32)
        return emb

    def _step(self, st, guidance_scale):
        """Device work of one denoising step on the static buffers ``st``."""
        lat, n = st['latents'], st['latents'].shape[0]
        eps = self.unet(torch.cat([lat, lat], dim=0), st['t'], st['emb'])
        eps_u, eps_c = eps[:n], eps[n:]
        eps = eps_u + guidance_scale * (eps_c - eps_u)
        lat.copy_((lat - 0.02 * eps).clamp_(-4, 4))
        st['stat'].copy_(eps.float().mean(dim=(1, 2, 3)))

    def _state(self, n, latent_h, latent_w, tokens):
        spec, dev = self.unet.spec, self.device
        key = (n, latent_h, latent_w, tuple(id(m.processor) for m in self._attn), tokens)
        st = self._graphs.get(key)
        if st is None:
            if len(self._graphs) > 4:
                self._graphs.clear()
            st = {
                'emb': torch.empty(2 * n, tokens, spec.cross_attention_dim, dtype=self.dtype, device=dev),
                'lat0': torch.empty(n, spec.in_channels, latent_h, latent_w, dtype=self.dtype, device=dev),
                'latents': torch.empty(n, spec.in_channels, latent_h, latent_w, dtype=self.dtype, device=dev),
                't': torch.zeros(1, dtype=torch.float32, device=dev),
                'stat': torch.zeros(n, dtype=torch.float32, device=dev),
                'graph': None, 'eager_steps': 0,
            }
            self._graphs[key] = st
        return st

    @torch.no_grad()
    def __call__(self, prompt=None, num_inference_steps: int = 50, generator: Optional[torch.Generator] = None,
                 callback=None, guidance_scale: float = 7.5, height: Optional[int] = None, width: Optional[int] = None,
                 negative_prompt=None, num_images_per_prompt: int = 1, prompt_embeds: Optional[torch.Tensor] = None,
                 negative_prompt_embeds: Optional[torch.Tensor] = None):
        """``height`` / ``width``: the image size in pixels, as diffusers takes it (default: the model's own square
        size); the latent is ``height // 8 x width // 8``. ``negative_prompt`` reaches ``check_inputs`` positionally, in
        diffusers' SD order; the synthetic encoder ignores all text, so it changes no embedding or random draw.
        ``num_images_per_prompt``: like diffusers, every prompt's embeddings are repeated prompt-major (the batch is
        ``[uncond x N x n, cond x N x n]``) and one latent is drawn per image; with 1 the draws are those of a call
        without it. ``prompt_embeds`` / ``negative_prompt_embeds`` ``[N, T, C]`` (``prompt=None``; e.g. ``T`` = 154
        or 231 for chunked long-prompt embeddings): the cond and uncond halves of the batch as given (zeros for a missing
        uncond half) instead of the synthetic encoder's draw; ``check_inputs`` gets ``prompt=None`` and them by name."""
        spec = self.unet.spec
        height = spec.sample_size * self.vae_scale_factor if height is None else height
        width = spec.sample_size * self.vae_scale_factor if width is None else width
        if prompt_embeds is not None:
            self.check_inputs(prompt, height, width, None, negative_prompt, prompt_embeds=prompt_embeds,
                              negative_prompt_embeds=negative_prompt_embeds)
        elif negative_prompt is None:
            self.check_inputs(prompt, height, width)
        else:
            self.check_inputs(prompt, height, width, None, negative_prompt)
        if prompt_embeds is not None:
            prompts = [None] * prompt_embeds.shape[0]
        else:
            prompts = [prompt] if isinstance(prompt, str) else list(prompt)
        latent_h, latent_w = height // self.vae_scale_factor, width // self.vae_scale_factor
        if generator is None:
            generator = torch.Generator().manual_seed(self.seed)
        cuda = self.device.type == 'cuda'
        if prompt_embeds is not None:
            cond = prompt_embeds.detach().float().cpu()
            uncond = torch.zeros_like(cond) if negative_prompt_embeds is None \
                else negative_prompt_embeds.detach().float().cpu()
            emb_h = torch.cat([uncond, cond]).to(self.dtype)
        else:
            emb_h = self.encode(prompts, generator).to(self.dtype)
        if num_images_per_prompt != 1:                        # [2, N, ...] -> [2, N * n, ...], each prompt n times
            emb_h = emb_h.view(2, len(prompts), *emb_h.shape[1:]).repeat_interleave(num_images_per_prompt, dim=1) \
                .reshape(-1, *emb_h.shape[1:])
        n = len(prompts) * num_images_per_prompt
        lat_h = torch.randn(n, spec.in_channels, latent_h, latent_w, generator=generator,
                            dtype=torch.float32).to(self.dtype)
        t_h = torch.tensor([[1000.0 * (1.0 - i / max(1, num_inference_steps))] for i in range(num_inference_steps)])
        out_h = torch.empty(n, dtype=torch.float32)
        if cuda:
            emb_h, lat_h, t_h, out_h = emb_h.pin_memory(), lat_h.pin_memory(), t_h.pin_memory(), out_h.pin_memory()
        self.h2d_bytes_per_step = emb_h.numel() * emb_h.element_size() + lat_h.numel() * lat_h.element_size() + 4
        self.d2h_bytes_per_step = n * 4
        st = self._state(n, latent_h, latent_w, emb_h.shape[1])
        for i in range(num_inference_steps):
            st['emb'].copy_(emb_h, non_blocking=True)            # H2D: the step's inputs
            st['lat0'].copy_(lat_h, non_blocking=True)
            st['t'].copy_(t_h[i], non_blocking=True)
            if i == 0:
                st['latents'].copy_(st['lat0'])
            if self.cuda_graph and st['graph'] is not None:
                st['graph'].replay()
            elif self.cuda_graph and st['eager_steps'] >= 1:
                graph = torch.cuda.CUDAGraph()
                with torch.cuda.graph(graph):
                    self._step(st, guidance_scale)
                st['graph'] = graph
                graph.replay()                                     # capture does not execute: run the step now
            else:
                self._step(st, guidance_scale)
                st['eager_steps'] += 1
            out_h.copy_(st['stat'], non_blocking=True)           # D2H: the step's result
            if callback is not None:
                callback(i, float(t_h[i]), st['latents'])
        latents = st['latents'].clone()
        image = latents[:, :3].float()
        images = self.image_processor.postprocess(image, output_type='pil')
        return SimpleNamespace(images=images, latents=latents)


def make_pipeline(spec: UNetSpec = SD21_SPEC, body: str = 'skeleton', dtype=torch.float32, device='cpu',
                  seed: int = 0, init_on_device: bool = False, cuda_graph: bool = False) -> SyntheticPipeline:
    """Random-init pipeline. Weights are drawn on the CPU from ``seed`` (identical on every box) unless
    ``init_on_device`` (fast for the full-size bodies; values then depend on the device RNG)."""
    gen_state = torch.random.get_rng_state()
    torch.manual_seed(seed)
    if init_on_device and torch.device(device).type == 'cuda':
        with torch.device(device):
            unet = SyntheticUNet(spec, body=body)
    else:
        unet = SyntheticUNet(spec, body=body)
    torch.random.set_rng_state(gen_state)
    return SyntheticPipeline(unet, dtype=dtype, device=device, seed=seed, cuda_graph=cuda_graph)


# ---------------------------------------------------------------------------------------------------------------
# Stable Diffusion 3: MM-DiT transformer with joint attention
# ---------------------------------------------------------------------------------------------------------------
class JointAttnProcessor:
    """The un-hooked joint attention: diffusers' ``JointAttnProcessor2_0`` op for op (image projections, optional
    q / k norms on ``[B, heads, N, d]``, context projections and their norms, concatenation image-then-context, one
    SDPA, split, ``to_add_out`` unless ``context_pre_only``, ``to_out``)."""

    def __call__(self, attn, hidden_states, encoder_hidden_states=None, attention_mask=None, *args, **kwargs):
        residual = hidden_states
        b = hidden_states.shape[0]
        query, key, value = attn.to_q(hidden_states), attn.to_k(hidden_states), attn.to_v(hidden_states)
        d = key.shape[-1] // attn.heads
        query = query.view(b, -1, attn.heads, d).transpose(1, 2)
        key = key.view(b, -1, attn.heads, d).transpose(1, 2)
        value = value.view(b, -1, attn.heads, d).transpose(1, 2)
        if attn.norm_q is not None:
            query = attn.norm_q(query)
        if attn.norm_k is not None:
            key = attn.norm_k(key)
        if encoder_hidden_states is not None:
            cq = attn.add_q_proj(encoder_hidden_states).view(b, -1, attn.heads, d).transpose(1, 2)
            ck = attn.add_k_proj(encoder_hidden_states).view(b, -1, attn.heads, d).transpose(1, 2)
            cv = attn.add_v_proj(encoder_hidden_states).view(b, -1, attn.heads, d).transpose(1, 2)
            if attn.norm_added_q is not None:
                cq = attn.norm_added_q(cq)
            if attn.norm_added_k is not None:
                ck = attn.norm_added_k(ck)
            query = torch.cat([query, cq], dim=2)
            key = torch.cat([key, ck], dim=2)
            value = torch.cat([value, cv], dim=2)
        hidden_states = F.scaled_dot_product_attention(query, key, value, dropout_p=0.0, is_causal=False)
        hidden_states = hidden_states.transpose(1, 2).reshape(b, -1, attn.heads * d).to(query.dtype)
        if encoder_hidden_states is not None:
            hidden_states, encoder_hidden_states = hidden_states[:, :residual.shape[1]], \
                hidden_states[:, residual.shape[1]:]
            if not attn.context_pre_only:
                encoder_hidden_states = attn.to_add_out(encoder_hidden_states)
        hidden_states = attn.to_out[1](attn.to_out[0](hidden_states))
        if encoder_hidden_states is not None:
            return hidden_states, encoder_hidden_states
        return hidden_states


class SyntheticJointAttention(nn.Module):
    """The attributes of diffusers' ``Attention`` that a joint block's processor reads."""

    def __init__(self, dim: int, heads: int, dim_head: int, qk_norm: bool, context_pre_only: bool):
        super().__init__()
        inner = heads * dim_head
        self.heads = heads
        self.scale = dim_head ** -0.5
        self.context_pre_only = context_pre_only
        self.to_q, self.to_k, self.to_v = (nn.Linear(dim, inner) for _ in range(3))
        self.add_q_proj, self.add_k_proj, self.add_v_proj = (nn.Linear(dim, inner) for _ in range(3))
        norm = (lambda: nn.RMSNorm(dim_head, eps=1e-6)) if qk_norm else (lambda: None)
        self.norm_q, self.norm_k, self.norm_added_q, self.norm_added_k = norm(), norm(), norm(), norm()
        self.to_out = nn.ModuleList([nn.Linear(inner, dim), nn.Dropout(0.0)])
        self.to_add_out = None if context_pre_only else nn.Linear(inner, dim)
        self.processor = JointAttnProcessor()

    def set_processor(self, processor):
        self.processor = processor

    def forward(self, hidden_states, encoder_hidden_states=None, attention_mask=None, **kwargs):
        return self.processor(self, hidden_states, encoder_hidden_states=encoder_hidden_states,
                              attention_mask=attention_mask, **kwargs)


class JointTransformerBlock(nn.Module):
    """An MM-DiT block: the joint attention over the normed image and context streams, then a feed-forward on each
    (none on the context after the ``context_pre_only`` last block)."""

    def __init__(self, dim, heads, dim_head, qk_norm, context_pre_only):
        super().__init__()
        self.context_pre_only = context_pre_only
        self.norm1 = nn.LayerNorm(dim)
        self.norm1_context = nn.LayerNorm(dim)
        self.attn = SyntheticJointAttention(dim, heads, dim_head, qk_norm, context_pre_only)
        self.ff = nn.Linear(dim, dim)
        self.ff_context = None if context_pre_only else nn.Linear(dim, dim)

    def forward(self, hidden_states, encoder_hidden_states, temb):
        x = self.norm1(hidden_states) + temb[:, None]
        attn_out, ctx_out = self.attn(x, encoder_hidden_states=self.norm1_context(encoder_hidden_states))
        hidden_states = hidden_states + attn_out
        hidden_states = hidden_states + self.ff(F.gelu(hidden_states))
        if self.context_pre_only:
            return None, hidden_states
        encoder_hidden_states = encoder_hidden_states + ctx_out
        return encoder_hidden_states + self.ff_context(F.gelu(encoder_hidden_states)), hidden_states


@dataclass
class SD3Spec:
    """Shape of an SD3 transformer: ``heads`` heads of ``dim_head`` in each of ``blocks`` joint blocks, a
    ``sample_size`` latent of ``in_channels`` cut into ``patch_size`` patches, and a context of 77 CLIP rows plus
    ``t5_rows`` T5 rows (``max_sequence_length``) of ``joint_attention_dim`` channels."""
    name: str
    sample_size: int
    blocks: int
    heads: int
    dim_head: int = 64
    patch_size: int = 2
    in_channels: int = 16
    joint_attention_dim: int = 4096
    t5_rows: int = 256
    qk_norm: bool = False


# public transformer/config.json shapes of stabilityai/stable-diffusion-3-medium-diffusers and
# stabilityai/stable-diffusion-3.5-large (RMS q / k norm), at their 1024-pixel (128 x 128 latent) size
SD3_MEDIUM_SPEC = SD3Spec('sd3-medium', 128, 24, 24)
SD35_LARGE_SPEC = SD3Spec('sd3.5-large', 128, 38, 38, qk_norm=True)
# small joint trees for the tests: RMS q / k norm, three blocks, a 16-row T5 context (93 rows in all)
TINY_SD3_SPEC = SD3Spec('tiny-sd3', 32, 3, 2, dim_head=32, in_channels=4, joint_attention_dim=64, t5_rows=16,
                        qk_norm=True)


class SyntheticSD3Transformer(nn.Module):
    """SD3Transformer2DModel-shaped random-init network: patchify, ``transformer_blocks`` of joint blocks (the last
    one ``context_pre_only``), unpatchify. ``forward(hidden_states=, encoder_hidden_states=, timestep=)`` returns a
    1-tuple, as diffusers' does with ``return_dict=False``."""

    def __init__(self, spec: SD3Spec):
        super().__init__()
        self.spec = spec
        dim = spec.heads * spec.dim_head
        self.config = SimpleNamespace(sample_size=spec.sample_size, patch_size=spec.patch_size,
                                      in_channels=spec.in_channels, joint_attention_dim=spec.joint_attention_dim)
        self.pos_embed = nn.Conv2d(spec.in_channels, dim, spec.patch_size, stride=spec.patch_size)
        self.time_proj = nn.Linear(1, dim)
        self.context_embedder = nn.Linear(spec.joint_attention_dim, dim)
        self.transformer_blocks = nn.ModuleList([
            JointTransformerBlock(dim, spec.heads, spec.dim_head, spec.qk_norm, i == spec.blocks - 1)
            for i in range(spec.blocks)])
        self.norm_out = nn.LayerNorm(dim)
        self.proj_out = nn.Linear(dim, spec.patch_size ** 2 * spec.in_channels)

    def forward(self, hidden_states, encoder_hidden_states, timestep, return_dict: bool = False):
        b, c, h, w = hidden_states.shape
        p = self.spec.patch_size
        x = self.pos_embed(hidden_states).flatten(2).transpose(1, 2)
        temb = self.time_proj(timestep.reshape(-1, 1).expand(b, 1).to(x.dtype) / 1000)
        ctx = self.context_embedder(encoder_hidden_states)
        for block in self.transformer_blocks:
            ctx, x = block(x, ctx, temb)
        x = self.proj_out(self.norm_out(x)).view(b, h // p, w // p, p, p, c)
        return (x.permute(0, 5, 1, 3, 2, 4).reshape(b, c, h, w),)


class SentencePieceTokenizer:
    """T5-tokenizer stand-in: whitespace words, case kept, each cut into pieces of at most 4 characters; a word's
    first piece carries sentencepiece's ``▁`` word-start marker (so ``'giraffe'`` is ``['▁gira', 'ffe']``)."""

    def tokenize(self, text: str) -> List[str]:
        out = []
        for word in text.split():
            pieces = [word[i:i + 4] for i in range(0, len(word), 4)]
            out += ['▁' + pieces[0]] + pieces[1:]
        return out


class SyntheticSD3Pipeline:
    """A StableDiffusion3Pipeline-shaped driver around :class:`SyntheticSD3Transformer`: ``transformer`` and no
    ``unet``, ``tokenizer`` (CLIP-style) and ``tokenizer_3`` (sentencepiece-style), ``check_inputs`` in diffusers'
    SD3 parameter order, ``image_processor.postprocess`` and a CFG loop over ``[uncond x N, cond x N]`` batches whose
    context is 77 CLIP rows then ``max_sequence_length`` T5 rows (seeded gaussian embeddings)."""

    def __init__(self, transformer: SyntheticSD3Transformer, dtype=torch.float32, device='cpu', seed: int = 0):
        self.transformer = transformer.to(device=device, dtype=dtype).eval()
        self.dtype, self.device = dtype, torch.device(device)
        self.vae_scale_factor = 8
        self.tokenizer = WhitespaceTokenizer()
        self.tokenizer_3 = SentencePieceTokenizer()
        self.image_processor = _ImageProcessor()
        self.seed = seed

    def check_inputs(self, prompt, prompt_2, prompt_3, height, width, negative_prompt=None, negative_prompt_2=None,
                     negative_prompt_3=None, prompt_embeds=None, negative_prompt_embeds=None, *args, **kwargs):
        if prompt is None and prompt_embeds is None:
            raise ValueError('Provide either `prompt` or `prompt_embeds`')
        if height % (self.vae_scale_factor * self.transformer.spec.patch_size) or \
                width % (self.vae_scale_factor * self.transformer.spec.patch_size):
            raise ValueError(f'`height` and `width` must be divisible by '
                             f'{self.vae_scale_factor * self.transformer.spec.patch_size}')

    @torch.no_grad()
    def __call__(self, prompt=None, prompt_2=None, prompt_3=None, height: Optional[int] = None,
                 width: Optional[int] = None, num_inference_steps: int = 28, guidance_scale: float = 7.0,
                 num_images_per_prompt: int = 1, generator: Optional[torch.Generator] = None,
                 max_sequence_length: Optional[int] = None):
        spec = self.transformer.spec
        height = spec.sample_size * self.vae_scale_factor if height is None else height
        width = spec.sample_size * self.vae_scale_factor if width is None else width
        self.check_inputs(prompt, prompt_2, prompt_3, height, width)
        prompts = [prompt] if isinstance(prompt, str) else list(prompt)
        rows = 77 + (spec.t5_rows if max_sequence_length is None else max_sequence_length)
        if generator is None:
            generator = torch.Generator().manual_seed(self.seed)
        n = len(prompts) * num_images_per_prompt
        emb = torch.randn(2, len(prompts), rows, spec.joint_attention_dim, generator=generator)
        emb = emb.repeat_interleave(num_images_per_prompt, dim=1).reshape(2 * n, rows, -1)
        lat = torch.randn(n, spec.in_channels, height // self.vae_scale_factor, width // self.vae_scale_factor,
                          generator=generator)
        emb, lat = emb.to(self.device, self.dtype), lat.to(self.device, self.dtype)
        for i in range(num_inference_steps):
            t = torch.full((2 * n,), 1000.0 * (1.0 - i / max(1, num_inference_steps)), device=self.device)
            eps = self.transformer(hidden_states=torch.cat([lat, lat]), encoder_hidden_states=emb, timestep=t,
                                   return_dict=False)[0]
            eps = eps[:n] + guidance_scale * (eps[n:] - eps[:n])
            lat = (lat - 0.02 * eps).clamp(-4, 4)
        images = self.image_processor.postprocess(lat[:, :3].float(), output_type='pil')
        return SimpleNamespace(images=images, latents=lat)


def make_sd3_pipeline(spec: SD3Spec = TINY_SD3_SPEC, dtype=torch.float32, device='cpu', seed: int = 0,
                      init_on_device: bool = False) -> SyntheticSD3Pipeline:
    """Random-init SD3-shaped pipeline; weights drawn on the CPU from ``seed`` unless ``init_on_device``."""
    gen_state = torch.random.get_rng_state()
    torch.manual_seed(seed)
    if init_on_device and torch.device(device).type == 'cuda':
        with torch.device(device):
            transformer = SyntheticSD3Transformer(spec)
    else:
        transformer = SyntheticSD3Transformer(spec)
    torch.random.set_rng_state(gen_state)
    return SyntheticSD3Pipeline(transformer, dtype=dtype, device=device, seed=seed)


# ---------------------------------------------------------------------------------------------------------------
# FLUX.1: MM-DiT with double-stream and single-stream blocks, packed latents and 3-axis RoPE
# ---------------------------------------------------------------------------------------------------------------
def flux_rotary_emb(x, freqs):
    """diffusers' ``apply_rotary_emb(x, (cos, sin), use_real=True, use_real_unbind_dim=-1)``: ``x`` ``[B, H, S, D]``,
    ``cos`` / ``sin`` ``[S, D]``; interleaved real / imaginary pairs, computed in fp32 and cast back."""
    cos, sin = freqs
    cos, sin = cos[None, None].to(x.device), sin[None, None].to(x.device)
    x_real, x_imag = x.reshape(*x.shape[:-1], -1, 2).unbind(-1)
    x_rotated = torch.stack([-x_imag, x_real], dim=-1).flatten(3)
    return (x.float() * cos + x_rotated.float() * sin).to(x.dtype)


class FluxAttnProcessor:
    """The un-hooked FLUX attention: diffusers' ``FluxAttnProcessor2_0`` op for op (image projections, q / k norms on
    ``[B, heads, N, d]``; with a context its projections and norms, concatenated context-then-image; RoPE on q and k;
    one SDPA; with a context the split, ``to_out`` and ``to_add_out``, else the attention output alone)."""

    def __call__(self, attn, hidden_states, encoder_hidden_states=None, attention_mask=None, image_rotary_emb=None):
        b = hidden_states.shape[0] if encoder_hidden_states is None else encoder_hidden_states.shape[0]
        query, key, value = attn.to_q(hidden_states), attn.to_k(hidden_states), attn.to_v(hidden_states)
        d = key.shape[-1] // attn.heads
        query = query.view(b, -1, attn.heads, d).transpose(1, 2)
        key = key.view(b, -1, attn.heads, d).transpose(1, 2)
        value = value.view(b, -1, attn.heads, d).transpose(1, 2)
        if attn.norm_q is not None:
            query = attn.norm_q(query)
        if attn.norm_k is not None:
            key = attn.norm_k(key)
        if encoder_hidden_states is not None:
            cq = attn.add_q_proj(encoder_hidden_states).view(b, -1, attn.heads, d).transpose(1, 2)
            ck = attn.add_k_proj(encoder_hidden_states).view(b, -1, attn.heads, d).transpose(1, 2)
            cv = attn.add_v_proj(encoder_hidden_states).view(b, -1, attn.heads, d).transpose(1, 2)
            if attn.norm_added_q is not None:
                cq = attn.norm_added_q(cq)
            if attn.norm_added_k is not None:
                ck = attn.norm_added_k(ck)
            query = torch.cat([cq, query], dim=2)
            key = torch.cat([ck, key], dim=2)
            value = torch.cat([cv, value], dim=2)
        if image_rotary_emb is not None:
            query = flux_rotary_emb(query, image_rotary_emb)
            key = flux_rotary_emb(key, image_rotary_emb)
        hidden_states = F.scaled_dot_product_attention(query, key, value, attn_mask=attention_mask, dropout_p=0.0,
                                                       is_causal=False)
        hidden_states = hidden_states.transpose(1, 2).reshape(b, -1, attn.heads * d).to(query.dtype)
        if encoder_hidden_states is None:
            return hidden_states
        encoder_hidden_states, hidden_states = hidden_states[:, :encoder_hidden_states.shape[1]], \
            hidden_states[:, encoder_hidden_states.shape[1]:]
        hidden_states = attn.to_out[1](attn.to_out[0](hidden_states))
        encoder_hidden_states = attn.to_add_out(encoder_hidden_states)
        return hidden_states, encoder_hidden_states


class SyntheticFluxAttention(nn.Module):
    """The attributes of diffusers' ``Attention`` as FLUX builds it (``qk_norm='rms_norm'``, ``bias=True``): a
    double-stream attention has the ``add_*_proj`` context projections, their norms, ``to_out`` and ``to_add_out``;
    a single-stream one (``pre_only``) has neither context projections nor ``to_out``."""

    def __init__(self, dim: int, heads: int, dim_head: int, double: bool):
        super().__init__()
        inner = heads * dim_head
        self.heads = heads
        self.scale = dim_head ** -0.5
        self.pre_only = not double
        self.to_q, self.to_k, self.to_v = (nn.Linear(dim, inner) for _ in range(3))
        self.norm_q, self.norm_k = nn.RMSNorm(dim_head, eps=1e-6), nn.RMSNorm(dim_head, eps=1e-6)
        if double:
            self.add_q_proj, self.add_k_proj, self.add_v_proj = (nn.Linear(dim, inner) for _ in range(3))
            self.norm_added_q, self.norm_added_k = nn.RMSNorm(dim_head, eps=1e-6), nn.RMSNorm(dim_head, eps=1e-6)
            self.to_out = nn.ModuleList([nn.Linear(inner, dim), nn.Dropout(0.0)])
            self.to_add_out = nn.Linear(inner, dim)
        else:
            self.add_q_proj = self.add_k_proj = self.add_v_proj = None
            self.norm_added_q = self.norm_added_k = None
        self.processor = FluxAttnProcessor()

    def set_processor(self, processor):
        self.processor = processor

    def forward(self, hidden_states, encoder_hidden_states=None, attention_mask=None, image_rotary_emb=None):
        return self.processor(self, hidden_states, encoder_hidden_states, attention_mask, image_rotary_emb)


class FluxTransformerBlock(nn.Module):
    """A double-stream block: the joint attention over the modulated image and context streams, then a feed-forward
    on each. Returns ``(encoder_hidden_states, hidden_states)`` as diffusers' does."""

    def __init__(self, dim, heads, dim_head):
        super().__init__()
        self.norm1 = nn.LayerNorm(dim, elementwise_affine=False, eps=1e-6)
        self.norm1_context = nn.LayerNorm(dim, elementwise_affine=False, eps=1e-6)
        self.attn = SyntheticFluxAttention(dim, heads, dim_head, double=True)
        self.ff = nn.Linear(dim, dim)
        self.ff_context = nn.Linear(dim, dim)

    def forward(self, hidden_states, encoder_hidden_states, temb, image_rotary_emb):
        x = self.norm1(hidden_states) + temb[:, None]
        c = self.norm1_context(encoder_hidden_states) + temb[:, None]
        attn_out, ctx_out = self.attn(hidden_states=x, encoder_hidden_states=c, image_rotary_emb=image_rotary_emb)
        hidden_states = hidden_states + attn_out
        hidden_states = hidden_states + self.ff(F.gelu(hidden_states))
        encoder_hidden_states = encoder_hidden_states + ctx_out
        encoder_hidden_states = encoder_hidden_states + self.ff_context(F.gelu(encoder_hidden_states))
        return encoder_hidden_states, hidden_states


class FluxSingleTransformerBlock(nn.Module):
    """A single-stream block on the joined ``[text, image]`` sequence: the attention (``pre_only``, no context
    argument) in parallel with an MLP, both through ``proj_out``."""

    def __init__(self, dim, heads, dim_head):
        super().__init__()
        self.norm = nn.LayerNorm(dim, elementwise_affine=False, eps=1e-6)
        self.proj_mlp = nn.Linear(dim, dim)
        self.attn = SyntheticFluxAttention(dim, heads, dim_head, double=False)
        self.proj_out = nn.Linear(2 * dim, dim)

    def forward(self, hidden_states, temb, image_rotary_emb):
        x = self.norm(hidden_states) + temb[:, None]
        mlp = F.gelu(self.proj_mlp(x), approximate='tanh')
        attn_out = self.attn(hidden_states=x, image_rotary_emb=image_rotary_emb)
        return hidden_states + self.proj_out(torch.cat([attn_out, mlp], dim=2))


class FluxPosEmbed(nn.Module):
    """diffusers' ``FluxPosEmbed``: per axis of the ``[S, 3]`` position ids, ``get_1d_rotary_pos_embed(dim, pos,
    theta, use_real=True, repeat_interleave_real=True)`` in float64, concatenated over the axes: ``(cos, sin)``,
    each fp32 ``[S, sum(axes_dim)]``."""

    def __init__(self, theta: int, axes_dim: Sequence[int]):
        super().__init__()
        self.theta, self.axes_dim = theta, tuple(axes_dim)

    def forward(self, ids):
        pos = ids.float()
        cos_out, sin_out = [], []
        for i, dim in enumerate(self.axes_dim):
            freqs = 1.0 / (self.theta ** (torch.arange(0, dim, 2, dtype=torch.float64, device=ids.device)[:dim // 2]
                                          / dim))
            freqs = torch.outer(pos[:, i].double(), freqs)
            cos_out.append(freqs.cos().repeat_interleave(2, dim=1).float())
            sin_out.append(freqs.sin().repeat_interleave(2, dim=1).float())
        return torch.cat(cos_out, dim=-1), torch.cat(sin_out, dim=-1)


@dataclass
class FluxSpec:
    """Shape of a FLUX.1 transformer: ``double`` double-stream and ``single`` single-stream blocks of ``heads`` heads
    of ``dim_head`` (RoPE axes ``axes_dim``, summing to ``dim_head``), packed latents of ``in_channels`` (4 x the VAE's
    channels), a T5 context of ``t5_rows`` rows (``max_sequence_length``) of ``joint_attention_dim`` channels and a
    ``sample_size`` latent by default (the image is 8 x that)."""
    name: str
    double: int
    single: int
    heads: int = 24
    dim_head: int = 128
    axes_dim: Sequence[int] = (16, 56, 56)
    in_channels: int = 64
    joint_attention_dim: int = 4096
    pooled_projection_dim: int = 768
    t5_rows: int = 512
    guidance_embeds: bool = True
    sample_size: int = 128


# public transformer/config.json shapes of black-forest-labs/FLUX.1-dev and FLUX.1-schnell; the pipelines' default
# max_sequence_length is 512 for dev and 256 for schnell, at the default 1024-pixel (128 x 128 latent) size
FLUX_DEV_SPEC = FluxSpec('flux.1-dev', 19, 38)
FLUX_SCHNELL_SPEC = FluxSpec('flux.1-schnell', 19, 38, t5_rows=256, guidance_embeds=False)
# a small tree for the tests: two double and three single blocks, 2 heads of 32 (RoPE axes 8 / 12 / 12), a 24-row T5
# context, 256-pixel images by default
TINY_FLUX_SPEC = FluxSpec('tiny-flux', 2, 3, heads=2, dim_head=32, axes_dim=(8, 12, 12), in_channels=16,
                          joint_attention_dim=64, pooled_projection_dim=32, t5_rows=24, sample_size=32)


class SyntheticFluxTransformer(nn.Module):
    """FluxTransformer2DModel-shaped random-init network: ``x_embedder`` on the packed latent ``[B, hw, C]``, the
    timestep / guidance / pooled embedding, ``context_embedder``, RoPE of ``cat(txt_ids, img_ids)``, the
    ``transformer_blocks``, then the ``single_transformer_blocks`` on ``cat([context, image])``, and the image tokens
    out. ``forward(hidden_states=, encoder_hidden_states=, pooled_projections=, timestep=, img_ids=, txt_ids=,
    guidance=)`` returns a 1-tuple, as diffusers' does with ``return_dict=False``."""

    def __init__(self, spec: FluxSpec):
        super().__init__()
        self.spec = spec
        dim = spec.heads * spec.dim_head
        self.config = SimpleNamespace(patch_size=1, in_channels=spec.in_channels, num_layers=spec.double,
                                      num_single_layers=spec.single, attention_head_dim=spec.dim_head,
                                      num_attention_heads=spec.heads, joint_attention_dim=spec.joint_attention_dim,
                                      pooled_projection_dim=spec.pooled_projection_dim,
                                      guidance_embeds=spec.guidance_embeds, axes_dims_rope=tuple(spec.axes_dim))
        self.pos_embed = FluxPosEmbed(10000, spec.axes_dim)
        self.time_proj = nn.Linear(1, dim)
        self.guidance_proj = nn.Linear(1, dim) if spec.guidance_embeds else None
        self.pooled_proj = nn.Linear(spec.pooled_projection_dim, dim)
        self.context_embedder = nn.Linear(spec.joint_attention_dim, dim)
        self.x_embedder = nn.Linear(spec.in_channels, dim)
        self.transformer_blocks = nn.ModuleList([FluxTransformerBlock(dim, spec.heads, spec.dim_head)
                                                 for _ in range(spec.double)])
        self.single_transformer_blocks = nn.ModuleList([FluxSingleTransformerBlock(dim, spec.heads, spec.dim_head)
                                                        for _ in range(spec.single)])
        self.norm_out = nn.LayerNorm(dim, elementwise_affine=False, eps=1e-6)
        self.proj_out = nn.Linear(dim, spec.in_channels)

    def forward(self, hidden_states, encoder_hidden_states=None, pooled_projections=None, timestep=None, img_ids=None,
                txt_ids=None, guidance=None, joint_attention_kwargs=None, return_dict: bool = False):
        hidden_states = self.x_embedder(hidden_states)
        dtype = hidden_states.dtype
        temb = self.time_proj(timestep.reshape(-1, 1).to(dtype))
        if self.guidance_proj is not None and guidance is not None:
            temb = temb + self.guidance_proj(guidance.reshape(-1, 1).to(dtype))
        temb = F.silu(temb + self.pooled_proj(pooled_projections))
        encoder_hidden_states = self.context_embedder(encoder_hidden_states)
        image_rotary_emb = self.pos_embed(torch.cat((txt_ids, img_ids), dim=0))
        for block in self.transformer_blocks:
            encoder_hidden_states, hidden_states = block(hidden_states, encoder_hidden_states, temb, image_rotary_emb)
        hidden_states = torch.cat([encoder_hidden_states, hidden_states], dim=1)
        for block in self.single_transformer_blocks:
            hidden_states = block(hidden_states, temb, image_rotary_emb)
        hidden_states = hidden_states[:, encoder_hidden_states.shape[1]:]
        return (self.proj_out(self.norm_out(hidden_states)),)


def flux_image_ids(height: int, width: int, device=None) -> torch.Tensor:
    """diffusers' ``FluxPipeline._prepare_latent_image_ids`` for a packed ``height x width`` token grid: ``[hw, 3]``
    with (0, row, column) per token, row-major."""
    ids = torch.zeros(height, width, 3, device=device)
    ids[..., 1] += torch.arange(height, device=device)[:, None]
    ids[..., 2] += torch.arange(width, device=device)[None, :]
    return ids.reshape(height * width, 3)


def flux_pack(latents: torch.Tensor) -> torch.Tensor:
    """diffusers' ``FluxPipeline._pack_latents``: ``[B, C, H, W]`` -> ``[B, (H/2)(W/2), 4C]`` in 2 x 2 patches."""
    b, c, h, w = latents.shape
    latents = latents.view(b, c, h // 2, 2, w // 2, 2).permute(0, 2, 4, 1, 3, 5)
    return latents.reshape(b, (h // 2) * (w // 2), c * 4)


def flux_unpack(latents: torch.Tensor, h: int, w: int) -> torch.Tensor:
    """The inverse of :func:`flux_pack` for a ``h x w`` token grid: ``[B, hw, 4C]`` -> ``[B, C, 2h, 2w]``."""
    b, _, c4 = latents.shape
    latents = latents.view(b, h, w, c4 // 4, 2, 2).permute(0, 3, 1, 4, 2, 5)
    return latents.reshape(b, c4 // 4, 2 * h, 2 * w)


class SyntheticFluxPipeline:
    """A FluxPipeline-shaped driver around :class:`SyntheticFluxTransformer`: ``transformer`` and no ``unet``,
    ``tokenizer`` (CLIP-style, for the pooled embedding) and ``tokenizer_2`` (sentencepiece-style, for the T5 context),
    ``check_inputs`` with diffusers' FLUX signature, called after the default size is filled in, and
    ``image_processor.postprocess``. There is no CFG: one transformer forward per step over the ``prompts x images``
    batch (prompt-major), with the guidance scale as an embedding input (dev) -- except that a negative prompt with
    ``true_cfg_scale > 1`` runs a second forward on the negative embeddings, as diffusers' true CFG does. Latents are
    packed in 2 x 2 patches; the scheduler is a plain flow-matching Euler step."""

    def __init__(self, transformer: SyntheticFluxTransformer, dtype=torch.float32, device='cpu', seed: int = 0):
        self.transformer = transformer.to(device=device, dtype=dtype).eval()
        self.dtype, self.device = dtype, torch.device(device)
        self.vae_scale_factor = 8
        self.default_sample_size = transformer.spec.sample_size
        self.tokenizer = WhitespaceTokenizer()
        self.tokenizer_2 = SentencePieceTokenizer()
        self.image_processor = _ImageProcessor()
        self.seed = seed

    def check_inputs(self, prompt, prompt_2, height, width, negative_prompt=None, negative_prompt_2=None,
                     prompt_embeds=None, negative_prompt_embeds=None, pooled_prompt_embeds=None,
                     negative_pooled_prompt_embeds=None, callback_on_step_end_tensor_inputs=None,
                     max_sequence_length=None):
        if prompt is None and prompt_embeds is None:
            raise ValueError('Provide either `prompt` or `prompt_embeds`')
        if prompt is not None and prompt_embeds is not None:
            raise ValueError('Cannot forward both `prompt` and `prompt_embeds`')
        if max_sequence_length is not None and max_sequence_length > 512:
            raise ValueError(f'`max_sequence_length` cannot be greater than 512 but is {max_sequence_length}')

    def _embeds(self, n: int, rows: int, generator: torch.Generator):
        spec = self.transformer.spec
        emb = torch.randn(n, rows, spec.joint_attention_dim, generator=generator)
        pooled = torch.randn(n, spec.pooled_projection_dim, generator=generator)
        return emb, pooled

    @torch.no_grad()
    def __call__(self, prompt=None, prompt_2=None, negative_prompt=None, negative_prompt_2=None,
                 true_cfg_scale: float = 1.0, height: Optional[int] = None, width: Optional[int] = None,
                 num_inference_steps: int = 28, guidance_scale: float = 3.5, num_images_per_prompt: int = 1,
                 generator: Optional[torch.Generator] = None, prompt_embeds: Optional[torch.Tensor] = None,
                 pooled_prompt_embeds: Optional[torch.Tensor] = None,
                 negative_prompt_embeds: Optional[torch.Tensor] = None, max_sequence_length: int = 512):
        """``max_sequence_length``: the T5 rows of the context (diffusers' default 512; the schnell pipeline is run
        with 256). ``prompt_embeds`` ``[N, T, 4096]`` (with ``pooled_prompt_embeds``) replace the synthetic encoder's
        draw."""
        spec = self.transformer.spec
        height = height or self.default_sample_size * self.vae_scale_factor
        width = width or self.default_sample_size * self.vae_scale_factor
        self.check_inputs(prompt, prompt_2, height, width, negative_prompt=negative_prompt,
                          negative_prompt_2=negative_prompt_2, prompt_embeds=prompt_embeds,
                          negative_prompt_embeds=negative_prompt_embeds, pooled_prompt_embeds=pooled_prompt_embeds,
                          max_sequence_length=max_sequence_length)
        if generator is None:
            generator = torch.Generator().manual_seed(self.seed)
        if prompt_embeds is not None:
            n_prompts = prompt_embeds.shape[0]
            emb = prompt_embeds.detach().float().cpu()
            pooled = torch.zeros(n_prompts, spec.pooled_projection_dim) if pooled_prompt_embeds is None \
                else pooled_prompt_embeds.detach().float().cpu()
        else:
            n_prompts = 1 if isinstance(prompt, str) else len(prompt)
            emb, pooled = self._embeds(n_prompts, max_sequence_length, generator)
        true_cfg = true_cfg_scale > 1 and (negative_prompt is not None or negative_prompt_embeds is not None)
        if true_cfg:
            neg, neg_pooled = self._embeds(n_prompts, emb.shape[1], generator)
            if negative_prompt_embeds is not None:
                neg = negative_prompt_embeds.detach().float().cpu()
        n = n_prompts * num_images_per_prompt
        rep = lambda t: t.repeat_interleave(num_images_per_prompt, dim=0).to(self.device, self.dtype)
        emb, pooled = rep(emb), rep(pooled)
        if true_cfg:
            neg, neg_pooled = rep(neg), rep(neg_pooled)
        lh, lw = 2 * (height // (2 * self.vae_scale_factor)), 2 * (width // (2 * self.vae_scale_factor))
        lat = torch.randn(n, spec.in_channels // 4, lh, lw, generator=generator)
        lat = flux_pack(lat).to(self.device, self.dtype)
        img_ids = flux_image_ids(lh // 2, lw // 2, self.device).to(self.dtype)
        txt_ids = torch.zeros(emb.shape[1], 3, device=self.device, dtype=self.dtype)
        guidance = torch.full((n,), guidance_scale, device=self.device, dtype=torch.float32) \
            if spec.guidance_embeds else None
        sigmas = [1.0 - i / num_inference_steps for i in range(num_inference_steps)] + [0.0]
        for i in range(num_inference_steps):
            t = torch.full((n,), sigmas[i], device=self.device, dtype=self.dtype)
            v = self.transformer(hidden_states=lat, timestep=t, guidance=guidance, pooled_projections=pooled,
                                 encoder_hidden_states=emb, txt_ids=txt_ids, img_ids=img_ids, return_dict=False)[0]
            if true_cfg:
                v_neg = self.transformer(hidden_states=lat, timestep=t, guidance=guidance,
                                         pooled_projections=neg_pooled, encoder_hidden_states=neg, txt_ids=txt_ids,
                                         img_ids=img_ids, return_dict=False)[0]
                v = v_neg + true_cfg_scale * (v - v_neg)
            lat = (lat + (sigmas[i + 1] - sigmas[i]) * v).clamp(-4, 4)
        image = flux_unpack(lat, lh // 2, lw // 2)[:, :3].float()
        images = self.image_processor.postprocess(image, output_type='pil')
        return SimpleNamespace(images=images, latents=lat)


def make_flux_pipeline(spec: FluxSpec = TINY_FLUX_SPEC, dtype=torch.float32, device='cpu', seed: int = 0,
                       init_on_device: bool = False) -> SyntheticFluxPipeline:
    """Random-init FLUX-shaped pipeline; weights drawn on the CPU from ``seed`` unless ``init_on_device``."""
    gen_state = torch.random.get_rng_state()
    torch.manual_seed(seed)
    if init_on_device and torch.device(device).type == 'cuda':
        with torch.device(device):
            transformer = SyntheticFluxTransformer(spec)
    else:
        transformer = SyntheticFluxTransformer(spec)
    torch.random.set_rng_state(gen_state)
    return SyntheticFluxPipeline(transformer, dtype=dtype, device=device, seed=seed)
