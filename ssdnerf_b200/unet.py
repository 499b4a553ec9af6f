"""`DenoisingUnetMod` -- the reference's 2-D UNet over triplane latents, executed by hand-written sm_90a kernels.

Plugin surface kept from the reference (lib/models/architecture/ddpm/denoising.py:12-216, modules.py:12-129):
constructor kwargs, `forward(x_t, t, label=None, concat_cond=None)` and the state-dict key layout (SURVEY.md
Appendix D) so released checkpoints load unchanged.  The nn.Module tree below only HOLDS parameters; compute goes
through `UNetEngine`, which packs the weights to fp16 once and issues the C-ABI kernels of include/ssdnerf_b200.h §4:
implicit-GEMM 3x3 / 1x1 convolutions and attention GEMMs on wgmma tensor cores, GroupNorm(+scale/shift)+SiLU,
softmax and layout glue as fused memory-bound kernels.  Forward semantics of the blocks the reference inherits from
mmgen 0.7.2 are restated per SURVEY.md Appendix B.  Inference only (no autograd through the engine).
"""
import math
from copy import deepcopy

import torch
import torch.nn as nn

from . import _lib as N
from . import unet_ops as U
from .registry import MODULES


_GN_GROUPS = [32]      # construction-time GroupNorm group count (norm_cfg.num_groups), set by DenoisingUnetMod.__init__


def _gn(c):
    return nn.GroupNorm(_GN_GROUPS[0], c, eps=1e-5)


class _ResBlockParams(nn.Module):
    """parameter container with the key layout of DenoisingResBlockMod (modules.py:51-110)"""

    def __init__(self, cin, cout, emb_ch, dropout=0.0):
        super().__init__()
        self.conv_1 = nn.Sequential(_gn(cin), nn.SiLU(), nn.Conv2d(cin, cout, 3, padding=1))
        self.norm_with_embedding = nn.Module()
        self.norm_with_embedding.norm = _gn(cout)
        self.norm_with_embedding.embedding_layer = nn.Sequential(nn.SiLU(), nn.Linear(emb_ch, 2 * cout))
        conv_2 = [nn.SiLU(), nn.Dropout(dropout), nn.Conv2d(cout, cout, 3, padding=1)] if dropout > 0 \
            else [nn.SiLU(), nn.Conv2d(cout, cout, 3, padding=1)]
        self.conv_2 = nn.Sequential(*conv_2)
        if cin != cout:
            self.shortcut = nn.Conv2d(cin, cout, 1)
        self.cin, self.cout = cin, cout
        nn.init.zeros_(self.conv_2[-1].weight)      # mmgen init_weights: last conv of every ResBlock is zero
        nn.init.zeros_(self.conv_2[-1].bias)


class _AttnParams(nn.Module):
    """MultiHeadAttentionMod (modules.py:12-26)"""

    def __init__(self, c, num_heads):
        super().__init__()
        self.norm = _gn(c)
        self.qkv = nn.Conv1d(c, 3 * c, 1)
        self.proj = nn.Conv1d(c, c, 1)
        self.c, self.num_heads = c, num_heads
        nn.init.zeros_(self.proj.weight)
        nn.init.zeros_(self.proj.bias)


class _DownParams(nn.Module):
    def __init__(self, c):
        super().__init__()
        self.downsample = nn.Conv2d(c, c, 3, 2, 1)
        self.c = c


class _UpParams(nn.Module):
    def __init__(self, c):
        super().__init__()
        self.conv = nn.Conv2d(c, c, 3, 1, 1)
        self.c = c


class _TimeEmbedding(nn.Module):
    """mmgen TimeEmbedding(embedding_mode='sin'): sinusoidal (cos | sin) -> Linear -> SiLU -> Linear"""

    def __init__(self, base, emb_ch):
        super().__init__()
        self.blocks = nn.Sequential(nn.Linear(base, emb_ch), nn.SiLU(), nn.Linear(emb_ch, emb_ch))
        self.base = base

    def forward(self, t):
        half = self.base // 2
        freqs = torch.exp(-math.log(10000) * torch.arange(half, dtype=torch.float32, device=t.device) / half)
        args = t[:, None].float() * freqs[None]
        return self.blocks(torch.cat([torch.cos(args), torch.sin(args)], dim=-1))


@MODULES.register_module()
class DenoisingUnetMod(nn.Module):
    """Same constructor signature as lib/models/architecture/ddpm/denoising.py:14-43 (groups must be 1)."""

    def __init__(self, image_size, in_channels=3, concat_cond_channels=0, base_channels=128, resblocks_per_downsample=3,
                 num_timesteps=1000, use_rescale_timesteps=True, dropout=0, embedding_channels=-1, num_classes=0,
                 channels_cfg=None, groups=1, norm_cfg=dict(type='GN', num_groups=32), act_cfg=dict(type='SiLU', inplace=False),
                 shortcut_kernel_size=1, use_scale_shift_norm=False, num_heads=4, time_embedding_mode='sin',
                 time_embedding_cfg=None, resblock_cfg=dict(type='DenoisingResBlockMod'),
                 attention_cfg=dict(type='MultiHeadAttentionMod'), downsample_conv=True, upsample_conv=True,
                 downsample_cfg=dict(type='DenoisingDownsampleMod'), upsample_cfg=dict(type='DenoisingUpsampleMod'),
                 attention_res=[16, 8], pretrained=None):
        super().__init__()
        unsupported = []
        if groups != 1: unsupported.append('groups != 1')
        if num_classes != 0: unsupported.append('class conditioning')
        if not use_scale_shift_norm: unsupported.append('use_scale_shift_norm=False')
        if shortcut_kernel_size != 1: unsupported.append('shortcut_kernel_size != 1')
        if not (downsample_conv and upsample_conv): unsupported.append('pool / bare-interpolate resampling')
        if norm_cfg.get('type') != 'GN': unsupported.append('norm other than GroupNorm')
        if act_cfg.get('type') != 'SiLU': unsupported.append('activation other than SiLU')
        if time_embedding_mode != 'sin': unsupported.append('time_embedding_mode != sin')
        if unsupported:
            raise NotImplementedError('ssdnerf_b200.DenoisingUnetMod covers the configurations the reference ships; unsupported: '
                                      + ', '.join(unsupported))
        if not isinstance(channels_cfg, (list, tuple)):
            raise ValueError(f'Only support list for `channels_cfg`, receive {type(channels_cfg)}')
        self.num_classes, self.num_timesteps, self.use_rescale_timesteps = num_classes, num_timesteps, use_rescale_timesteps
        self.num_groups = int(norm_cfg.get('num_groups', 32))
        _GN_GROUPS[0] = self.num_groups
        self.out_channels = in_channels
        self.in_channels = in_channels
        self.concat_cond_channels = concat_cond_channels
        if isinstance(image_size, int):
            image_size = [image_size, image_size]
        assert len(image_size) == 2, 'The length of `image_size` should be 2.'
        self.image_size = list(image_size)
        self.channel_factor_list = list(channels_cfg)
        self.num_heads = num_heads
        self.base_channels = base_channels
        self.dropout = float(dropout)
        emb_ch = base_channels * 4 if embedding_channels == -1 else embedding_channels
        self.embedding_channels = emb_ch
        self.time_embedding = _TimeEmbedding(base_channels, emb_ch)

        attention_scale = [min(image_size) // int(res) for res in attention_res]
        scale = 1
        self.in_blocks = nn.ModuleList([nn.Sequential(nn.Conv2d(in_channels + concat_cond_channels, base_channels, 3, 1, padding=1))])
        self.in_channels_list = [base_channels]
        cin = base_channels
        for level, factor in enumerate(self.channel_factor_list):
            cin = base_channels if level == 0 else base_channels * self.channel_factor_list[level - 1]
            cout = base_channels * factor
            for _ in range(resblocks_per_downsample):
                layers = [_ResBlockParams(cin, cout, emb_ch, dropout)]
                cin = cout
                if scale in attention_scale:
                    layers.append(_AttnParams(cin, num_heads))
                self.in_channels_list.append(cin)
                self.in_blocks.append(nn.Sequential(*layers))
            if level != len(self.channel_factor_list) - 1:
                self.in_blocks.append(nn.Sequential(_DownParams(cin)))
                self.in_channels_list.append(cin)
                scale *= 2
        self.mid_blocks = nn.Sequential(_ResBlockParams(cin, cin, emb_ch, dropout), _AttnParams(cin, num_heads),
                                        _ResBlockParams(cin, cin, emb_ch, dropout))
        in_list = deepcopy(self.in_channels_list)
        self.out_blocks = nn.ModuleList()
        for level, factor in enumerate(self.channel_factor_list[::-1]):
            for idx in range(resblocks_per_downsample + 1):
                layers = [_ResBlockParams(cin + in_list.pop(), base_channels * factor, emb_ch, dropout)]
                cin = base_channels * factor
                if scale in attention_scale:
                    layers.append(_AttnParams(cin, num_heads))
                if level != len(self.channel_factor_list) - 1 and idx == resblocks_per_downsample:
                    layers.append(_UpParams(cin))
                    scale //= 2
                self.out_blocks.append(nn.Sequential(*layers))
        self.out = nn.Module()
        self.out.conv = nn.Conv2d(cin, in_channels, 3, padding=1)       # mmcv ConvModule registers conv before the norm
        self.out.gn = _gn(cin)
        _GN_GROUPS[0] = 32
        self._engine = None
        self._engine_key = None

    # ------------------------------------------------------------------ reference-facing API
    def engine(self, batch, device=None, hw=None):
        """(re)build the native engine for a batch size and latent size hw = (H, W) (default: image_size); weights are re-packed when
        parameters changed"""
        device = device or next(self.parameters()).device
        hw = tuple(int(v) for v in (hw if hw is not None else self.image_size))
        key = (batch, str(device), hw, tuple(p._version for p in self.parameters()))
        if self._engine is None or self._engine_key != key:
            old = self._engine
            self._engine = UNetEngine(self, batch, device, hw)
            if old is not None and self._engine_key is not None and self._engine_key[:3] == key[:3]:
                self._engine.bufs = old.bufs          # only the weights changed (optimizer step): keep the activation / scratch arena
            self._engine_key = key
        return self._engine

    def refresh_weights(self):
        """Drop the packed fp16 weights (and with them every captured DDIM graph keyed on this engine).  The caches follow
        `Parameter._version`, which `load_state_dict` / optimizers / in-place ops bump; writes through `.data` (e.g. an EMA hook doing
        `p.data.lerp_()`) do NOT -- call this after such an update."""
        self._engine = None
        self._engine_key = None

    def embedding(self, t):
        if self.use_rescale_timesteps:
            t = t.float() * (1000.0 / self.num_timesteps)
        return self.time_embedding(t)

    def forward(self, x_t, t, label=None, concat_cond=None, return_noise=False):
        """denoising.py:191-216. x_t [B,C,H,W] float; t [B] long. Returns fp32 [B,C,H,W].
        Differentiable: when autograd is recording the forward keeps its activations (save mode) and `backward` walks them with the
        hand-written passes -- frozen parameters + x_t requiring a gradient: input-gradient pass only (`UNetEngine.backward_nhwc`);
        any parameter requiring a gradient (training): input- and weight-gradient pass in one walk (`unet_train._UNetFullGrad`)."""
        if label is not None:
            raise NotImplementedError('class-conditional embedding is not built (num_classes == 0 in every reference config)')
        N.require_cuda(x_t)
        h = x_t
        if self.concat_cond_channels > 0:
            h = torch.cat([h, concat_cond], dim=1)
        B = h.shape[0]
        if t.dim() == 0 or t.numel() != B:
            t = t.expand(B)
        if torch.is_grad_enabled() and any(p.requires_grad for p in self.parameters()):
            # training of the denoiser: input-gradient + weight-gradient pass (unet_train.py)
            from .unet_train import forward_with_weight_grads
            return forward_with_weight_grads(self, h, t)
        if torch.is_grad_enabled() and h.requires_grad:
            if self.concat_cond_channels > 0:
                raise NotImplementedError('input gradients with concat_cond are not built (unused by the shipped configs)')
            return _UNetInputGrad.apply(h, self, t)
        with torch.no_grad():
            eng = self.engine(B, h.device, h.shape[-2:])
            eng.set_embedding(self.embedding(t.to(h.device)))
            v = eng.forward_nchw(h.float().contiguous())
            return v.permute(0, 3, 1, 2)[:, :self.out_channels].contiguous()


class _UNetInputGrad(torch.autograd.Function):
    """v = UNet(x_t, t) with d v / d x_t by the native input-gradient pass (frozen weights: guidance / val_optim never train them;
    training goes through unet_train._UNetFullGrad)."""

    @staticmethod
    def forward(ctx, x_t, module, t):
        B = x_t.shape[0]
        eng = module.engine(B, x_t.device, x_t.shape[-2:])
        eng.set_embedding(module.embedding(t.to(x_t.device)))
        eng.load_input_nchw(x_t.detach().float().contiguous())
        v = eng.forward_nhwc(save=True)
        ctx.eng, ctx.token, ctx.C = eng, eng.fwd_token, module.out_channels
        return v.permute(0, 3, 1, 2)[:, :module.out_channels].contiguous()

    @staticmethod
    def backward(ctx, grad_v):
        eng = ctx.eng
        if eng.fwd_token != ctx.token:
            raise RuntimeError('UNet input gradient: the engine ran another forward before this backward (activations overwritten)')
        return eng.backward_nchw(grad_v.contiguous().float()), None, None


def unet_widths(m):
    return sorted({m.base_channels * f for f in m.channel_factor_list} | {m.base_channels})


def is_narrow(m):
    """widths that are not all multiples of 64 (the tiled-triplane config: 80 / 160 / 320) run on the narrow-channel GEMM family"""
    return any(w % 64 for w in unet_widths(m))


class UNetEngine:
    """Packed fp16 weights + activation arena + launch sequence for one batch size and latent size.

    Channel widths must be multiples of 16 and divisible by the GroupNorm group count.  Widths that are all multiples of 64 (every
    paper config) use the default GEMM family; otherwise (`narrow`: the tiled-triplane config's 80 / 160 / 320 channels, GroupNorm(16),
    40 / 80-wide heads over 6 x 128 x 384 latents) every GEMM runs on the narrow-channel family (unet_ops, csrc/gemm_tc.cu algo 3),
    attention takes the unfused composition, the input is padded to 16 channels instead of 64, and the weight-gradient pass is not
    built (unet_train.WeightGradPass raises)."""

    CPAD_IN = 64

    def __init__(self, m: DenoisingUnetMod, batch, device, hw=None):
        self.m, self.B, self.dev = m, batch, torch.device(device)
        widths = unet_widths(m)
        self.groups = m.num_groups
        if any(w % 16 for w in widths) or any(w % self.groups for w in widths):
            raise NotImplementedError(f'native UNet engine: channel widths must be multiples of 16 and of the GroupNorm group count; got '
                                      f'widths {widths}, {self.groups} groups')
        self.narrow = is_narrow(m)
        attn_widths = sorted({p.c for p in m.modules() if isinstance(p, _AttnParams)})
        if any(c % m.num_heads or (c // m.num_heads) % 8 for c in attn_widths):
            raise NotImplementedError(f'native UNet engine: attention head widths must be multiples of 8; got widths {attn_widths} over '
                                      f'{m.num_heads} heads')
        self.H, self.W = (int(v) for v in (hw if hw is not None else m.image_size))
        self.bufs = {}
        self.cin_total = m.in_channels + m.concat_cond_channels
        if self.narrow:       # the input convolution's K: the channels rounded up to wgmma's 16-element K step, not to 64
            self.CPAD_IN = max(16, (self.cin_total + 15) // 16 * 16)
        assert self.cin_total <= self.CPAD_IN
        nw = self.narrow
        dev = self.dev
        f32 = lambda p: p.detach().float().contiguous().to(dev)
        # ---- op list + packed weights
        self.ops = []            # (kind, params dict)
        self.res_blocks = []     # for the scale/shift table
        self.n_norm = 0

        def res(p):
            d = dict(cin=p.cin, cout=p.cout, g1=f32(p.conv_1[0].weight), b1=f32(p.conv_1[0].bias),
                     w1=U.pack_conv_weight(p.conv_1[2].weight, narrow=nw).to(dev), c1b=f32(p.conv_1[2].bias),
                     g2=f32(p.norm_with_embedding.norm.weight), b2=f32(p.norm_with_embedding.norm.bias),
                     w2=U.pack_conv_weight(p.conv_2[-1].weight, narrow=nw).to(dev), c2b=f32(p.conv_2[-1].bias),
                     emb_w=f32(p.norm_with_embedding.embedding_layer[1].weight), emb_b=f32(p.norm_with_embedding.embedding_layer[1].bias),
                     n1=self._norm_slot(), n2=self._norm_slot(), idx=len(self.res_blocks), mod=p)
            if hasattr(p, 'shortcut'):
                d['ws'] = U.pack_linear_weight(p.shortcut.weight, narrow=nw).to(dev)
                d['wsb'] = f32(p.shortcut.bias)
            self.res_blocks.append(d)
            return ('res', d)

        def attn(p):
            return ('attn', dict(c=p.c, heads=p.num_heads, g=f32(p.norm.weight), b=f32(p.norm.bias),
                                 wqkv=U.pack_linear_weight(p.qkv.weight, narrow=nw).to(dev), bqkv=f32(p.qkv.bias),
                                 wproj=U.pack_linear_weight(p.proj.weight, narrow=nw).to(dev), bproj=f32(p.proj.bias), n=self._norm_slot(),
                                 mod=p))

        def layer(p):
            if isinstance(p, _ResBlockParams): return res(p)
            if isinstance(p, _AttnParams): return attn(p)
            if isinstance(p, _DownParams):
                return ('down', dict(c=p.c, w=U.pack_conv_weight(p.downsample.weight, narrow=nw).to(dev), b=f32(p.downsample.bias), mod=p))
            if isinstance(p, _UpParams):
                return ('up', dict(c=p.c, w=U.pack_upconv_weight(p.conv.weight, narrow=nw).to(dev), b=f32(p.conv.bias), mod=p))
            raise TypeError(type(p))

        conv_in = m.in_blocks[0][0]
        self.conv_in = dict(w=U.pack_conv_weight(conv_in.weight, cin_pad=self.CPAD_IN).to(dev), b=f32(conv_in.bias), cout=conv_in.out_channels)
        self.in_seq = [[layer(p) for p in blk] for blk in list(m.in_blocks)[1:]]
        self.mid_seq = [layer(p) for p in m.mid_blocks]
        self.out_seq = [[layer(p) for p in blk] for blk in m.out_blocks]
        self.out_norm = dict(g=f32(m.out.gn.weight), b=f32(m.out.gn.bias), n=self._norm_slot(), c=m.out.gn.num_channels)
        self.out_conv = dict(w=U.pack_conv_weight(m.out.conv.weight, narrow=nw).to(dev), b=f32(m.out.conv.bias), cout=m.out.conv.out_channels)
        # ---- GroupNorm quad-statistics arena: one [B, C/4, 2] slice per tensor that feeds a norm, filled by the producing GEMM's
        #      epilogue; zeroed once per forward (a single memset node in the captured graph)
        self.qarena = torch.zeros(4 * 1024 * 1024, dtype=torch.float32, device=dev)
        self.qoff = 0
        self.qslots = {}
        self._legacy_idx = 0
        self.ss_offsets, off = [], 0
        for d in self.res_blocks:
            self.ss_offsets.append(off)
            off += 2 * d['cout']
        self.ss_total = off
        self.ss_cur = torch.zeros(batch, self.ss_total, dtype=torch.float32, device=dev)
        self.saving, self.tape, self.fwd_token, self._bwd_packed = False, [], 0, False
        self.drop_p, self._drop_seed = float(m.dropout), None      # ResBlock dropout: active only in the training forward
        self.x_in = torch.zeros(batch, self.H, self.W, self.CPAD_IN, dtype=torch.float16, device=dev)
        self.v_out = torch.zeros(batch, self.H, self.W, self.out_conv['cout'], dtype=torch.float32, device=dev)

    def _norm_slot(self):
        self.n_norm += 1
        return self.n_norm - 1

    def _buf(self, key, shape, dtype=torch.float16):
        t = self.bufs.get(key)
        if t is None or tuple(t.shape) != tuple(shape) or t.dtype != dtype:
            t = torch.empty(*shape, dtype=dtype, device=self.dev)
            self.bufs[key] = t
        return t

    # ------------------------------------------------------------------ embeddings
    def scale_shift_rows(self, emb, live=False):
        """emb [R, emb_ch] -> [R, ss_total]: every ResBlock's Linear(SiLU(emb)) (NormWithEmbedding.embedding_layer).
        live=True uses the module's parameters themselves (differentiable: the weight-gradient pass back-propagates through it)."""
        e = torch.nn.functional.silu(emb.float())
        if live:
            lins = [d['mod'].norm_with_embedding.embedding_layer[1] for d in self.res_blocks]
            return torch.cat([torch.nn.functional.linear(e, l.weight.float(), l.bias.float()) for l in lins], dim=1)
        return torch.cat([torch.nn.functional.linear(e, d['emb_w'], d['emb_b']) for d in self.res_blocks], dim=1)

    def new_dropout_seed(self, training):
        """draw the dropout seed of the next save-mode forward from torch's CPU generator (None: dropout off)"""
        self._drop_seed = int(torch.randint(0, 2 ** 62, (1,)).item()) if (training and self.drop_p > 0) else None

    def _dropout(self, a2, block_idx):
        if self._drop_seed is not None:
            U.dropout_f16(a2, self._drop_seed + 0x9E3779B97F4A7C15 * (block_idx + 1), self.drop_p)

    def set_embedding(self, emb):
        """per-sample time embedding [B, emb_ch] for the next forward"""
        self.ss_cur.copy_(self.scale_shift_rows(emb))

    # ------------------------------------------------------------------ kernels
    def _q(self, key, channels):
        """quad-statistics slice [B, C/4, 2] for the tensor produced at `key` (stable across forwards: graph-capturable); None where a
        GroupNorm group of this tensor is not a whole number of quads (GroupNorm(16) over 80 / 160 channels): its producer then emits
        no statistics and the norm takes the separate statistics pass"""
        if (channels // self.groups) % 4:
            return None
        t = self.qslots.get(key)
        if t is None:
            n = self.B * (channels // 4) * 2
            t = self.qarena[self.qoff:self.qoff + n].view(self.B, channels // 4, 2)
            self.qoff += (n + 63) // 64 * 64
            assert self.qoff <= self.qarena.numel()
            self.qslots[key] = t
        return t

    def _gn(self, x1, q1, x2, q2, gamma, beta, out, silu, ss_off=None):
        """GroupNorm(self.groups) over the channel concat of x1 (+x2) from the quad statistics their producers emitted.
        Leaves the statistics descriptor the backward needs in `self._last_stats` = (is_quad, stats1, stats2)."""
        B, H, W, C1 = x1.shape
        C2 = x2.shape[-1] if x2 is not None else 0
        G = self.groups
        L, s = N.lib(), N.stream_ptr()
        ss = None
        if ss_off is not None:
            ss = N.c_void_p(self.ss_cur.data_ptr() + 4 * ss_off)
        if ((C1 + C2) // G) % 4 != 0 or q1 is None or (x2 is not None and q2 is None):
            # a group is not a whole number of 4-channel quads (sub-128-channel toy configs; GroupNorm(16) over 80 / 160 / 240 / 480
            # channels), or the producer could not emit quad statistics: separate statistics pass over group sums
            self._legacy_idx += 1          # one slot per call site, in call order (stable across forwards)
            st = self._q(('legacy', self._legacy_idx), G * 4)      # [B, G, 2], contiguous
            N.check(L.ssdnerf_gn_stats(N.ptr(x1), N.c_u32(C1), N.ptr(x2), N.c_u32(C2), N.c_u32(B), N.c_u32(H * W), N.c_u32(G), N.ptr(st), s))
            N.check(L.ssdnerf_gn_apply(N.ptr(x1), N.c_u32(C1), N.ptr(x2), N.c_u32(C2), N.c_u32(B), N.c_u32(H * W), N.c_u32(G), N.ptr(st),
                                       N.ptr(gamma), N.ptr(beta), ss, N.c_longlong(self.ss_total), N.c_f32(1e-5), N.c_int(int(silu)),
                                       N.ptr(out), s))
            self._last_stats = (False, st, None)
            return out
        self._last_stats = (True, q1, q2)
        N.check(L.ssdnerf_gn_apply_q(N.ptr(x1), N.c_u32(C1), N.ptr(x2), N.c_u32(C2), N.c_u32(B), N.c_u32(H * W), N.c_u32(G), N.ptr(q1),
                                     N.ptr(q2), N.ptr(gamma), N.ptr(beta), ss, N.c_longlong(self.ss_total), N.c_f32(1e-5),
                                     N.c_int(int(silu)), N.ptr(out), s))
        return out

    def _res(self, d, x, skip, tag):
        """x, skip: (tensor, quad-stats) pairs; returns the block output with the stats its epilogue emitted"""
        (x, qx), (sk, qs) = x, (skip if skip is not None else (None, None))
        B, H, W, _ = x.shape
        cin, cout = d['cin'], d['cout']
        nw = self.narrow
        if 'ws' in d:
            sc = U.conv3x3_f16(x, d['ws'].unsqueeze(0), cout, bias=d['wsb'], x2=sk, taps=1, out=self._buf(('sc', H, cout), (B, H, W, cout)),
                               narrow=nw)
        else:
            if sk is not None:      # an identity shortcut over a channel concat would need the concatenated tensor (mmgen adds it whole);
                raise NotImplementedError('ResBlock with a skip concat but no shortcut convolution (cin + skip == cout) is not built')
            sc = x
        qh1 = self._q(('h1', tag), cout)
        qo = self._q(('res_out', tag), cout)
        a = self._gn(x, qx, sk, qs, d['g1'], d['b1'], self._buf(('a', H, cin), (B, H, W, cin)), True)
        st1 = self._last_stats
        # saving keeps what the input-gradient pass re-reads (raw inputs of both GroupNorms + their statistics): h1 in a buffer of its own
        h1 = U.conv3x3_f16(a, d['w1'], cout, bias=d['c1b'], out=self._buf(('h1', tag) if self.saving else ('h1', H, cout), (B, H, W, cout)),
                           qstats=qh1, narrow=nw)
        a2 = self._gn(h1, qh1, None, None, d['g2'], d['b2'], self._buf(('a2', H, cout), (B, H, W, cout)), True, self.ss_offsets[d['idx']])
        st2 = self._last_stats
        if self.saving:
            self._dropout(a2, d['idx'])
        out = U.conv3x3_f16(a2, d['w2'], cout, bias=d['c2b'], residual=sc, out=self._buf(('res_out', tag), (B, H, W, cout)), qstats=qo,
                            narrow=nw)
        if self.saving:
            self.tape.append(dict(kind='res', d=d, x=x, sk=sk, st1=st1, h1=h1, st2=st2, out=out, tag=tag))
        return out, qo

    def _attn(self, d, x, tag):
        x, qx = x
        B, H, W, c = x.shape
        T, heads = H * W, d['heads']
        ch = c // heads
        L, s = N.lib(), N.stream_ptr()
        xn = self._gn(x, qx, None, None, d['g'], d['b'], self._buf(('xn', T, c), (B, H, W, c)), False)
        st = self._last_stats
        qkv = U.linear_f16(xn.view(B * T, c), d['wqkv'], bias=d['bqkv'], n=3 * c,
                           out=self._buf(('qkv', tag) if self.saving else ('qkv', T, c), (B * T, 3 * c)), narrow=self.narrow)
        o = self._attn_core(qkv, B, T, c, heads, ('o', T, c))
        # the projection's epilogue emits per-image quad statistics when an image is a whole number of 64-row tile halves; otherwise
        # (T = 48 at the tiled config's 4 x 12 level) the next GroupNorm takes the separate statistics pass
        qo = self._q(('attn_out', tag), c) if T % 64 == 0 else None
        out = U.linear_f16(o.view(B * T, c), d['wproj'], bias=d['bproj'], residual=x.view(B * T, c), n=c,
                           out=self._buf(('attn_out', tag), (B * T, c)), qstats=qo, stats_hw=T, narrow=self.narrow).view(B, H, W, c)
        if self.saving:
            self.tape.append(dict(kind='attn', d=d, x=x, st=st, qkv=qkv.view(B, T, 3 * c), out=out, tag=tag))
        return out, qo

    def _attn_core(self, qkv, B, T, c, heads, out_key):
        """softmax(q k^T / sqrt(ch)) v on the qkv projection [B*T, 3c] (legacy head layout) -> [B, T, c]"""
        ch = c // heads
        L, s = N.lib(), N.stream_ptr()
        if ch in (64, 128) and T % 64 == 0:
            return U.flash_attn(qkv.view(B, T, 3 * c), heads, 1.0 / math.sqrt(ch), out=self._buf(out_key, (B, T, c)))
        # unfused composition (scores -> softmax -> P V), kept for head widths / lengths the fused kernel does not cover
        S = U.attn_scores(qkv.view(B, T, 3 * c), heads, scale=1.0 / math.sqrt(ch), out=self._buf(('S', T), (B, heads, T, T), torch.float32),
                          narrow=self.narrow)
        P = self._buf(('P', T), (B, heads, T, T))
        N.check(L.ssdnerf_softmax_rows(N.ptr(S), N.c_u32(B * heads * T), N.c_u32(T), N.ptr(P), s))
        vt = self._buf(('vt', T, c), (B, heads, ch, T))
        N.check(L.ssdnerf_transpose_v(N.ptr(qkv), N.c_u32(B), N.c_u32(T), N.c_u32(heads), N.c_u32(ch), N.ptr(vt), s))
        return U.attn_pv(P, vt, out=self._buf(out_key, (B, T, c)), narrow=self.narrow)

    def _down(self, d, x, tag):
        x, _ = x
        B, H, W, c = x.shape
        qo = self._q(('down_out', tag), c)
        # stride-2 convolution straight from x: TMA boxes traverse every second pixel (no im2col buffer)
        out = U.conv3x3_s2_f16(x, d['w'], c, bias=d['b'], out=self._buf(('down_out', tag), (B, H // 2, W // 2, c)), qstats=qo, narrow=self.narrow)
        if self.saving:
            self.tape.append(dict(kind='down', d=d, x=x, out=out, tag=tag))
        return out, qo

    def _up(self, d, x, tag):
        x, _ = x
        B, H, W, c = x.shape
        qo = self._q(('up_out', tag), c)
        # nearest x2 + conv3x3 as four 2x2-tap phase convolutions of the low-resolution tensor (no upsampled buffer, 4/9 of the flops)
        out = U.upconv3x3_f16(x, d['w'], c, bias=d['b'], out=self._buf(('up_out', tag), (B, 2 * H, 2 * W, c)), qstats=qo, narrow=self.narrow)
        if self.saving:
            self.tape.append(dict(kind='up', d=d, x=x, out=out, tag=tag))
        return out, qo

    def _run(self, layers, h, skip, tag):
        for li, (kind, d) in enumerate(layers):
            t = (tag, li)
            if kind == 'res':
                h = self._res(d, h, skip, t)
                skip = None
            elif kind == 'attn':
                h = self._attn(d, h, t)
            elif kind == 'down':
                h = self._down(d, h, t)
            elif kind == 'up':
                h = self._up(d, h, t)
        return h

    # ------------------------------------------------------------------ forward
    def forward_nhwc(self, save=False):
        """x_in (self.x_in, fp16 NHWC padded) -> self.v_out (fp32 NHWC); all launches on the current stream, capture-safe.
        save=True keeps every tensor the input-gradient pass re-reads (per-layer buffers instead of shared scratch) and records the tape."""
        self.saving, self.tape = bool(save), []
        self.fwd_token += 1
        self.qarena[:max(self.qoff, 1)].zero_()
        self._legacy_idx = 0
        q0 = self._q(('conv_in',), self.conv_in['cout'])
        h = (U.conv3x3_f16(self.x_in, self.conv_in['w'], self.conv_in['cout'], bias=self.conv_in['b'],
                           out=self._buf(('conv_in',), (self.B, self.H, self.W, self.conv_in['cout'])), qstats=q0, narrow=self.narrow), q0)
        if self.saving:
            self.tape.append(dict(kind='conv_in', out=h[0]))
        hs = [h]
        for i, layers in enumerate(self.in_seq):
            h = self._run(layers, h, None, ('in', i))
            hs.append(h)
        h = self._run(self.mid_seq, h, None, ('mid',))
        for j, layers in enumerate(self.out_seq):
            h = self._run(layers, h, hs.pop(), ('out', j))
        h, qh = h
        B, H, W, c = h.shape
        a = self._gn(h, qh, None, None, self.out_norm['g'], self.out_norm['b'], self._buf(('a', H, c), (B, H, W, c)), True)
        if self.saving:
            self.tape.append(dict(kind='out', x=h, st=self._last_stats))
        U.conv3x3_f16(a, self.out_conv['w'], self.out_conv['cout'], bias=self.out_conv['b'], out=self.v_out, narrow=self.narrow)
        self.saving = False
        return self.v_out

    # ------------------------------------------------------------------ input-gradient pass (+ weight-gradient hooks: unet_train.py)
    def _pack_backward_weights(self):
        """transposed / tap-flipped fp16 copies of every weight, packed on first use (guidance and val_optim only)"""
        m, dev, nw = self.m, self.dev, self.narrow

        def params(seq, mods):
            for (kind, d), p in zip(seq, mods):
                if kind == 'res':
                    d['w1T'] = U.pack_conv_weight_dgrad(p.conv_1[2].weight, narrow=nw).to(dev)
                    d['w2T'] = U.pack_conv_weight_dgrad(p.conv_2[-1].weight, narrow=nw).to(dev)
                    if hasattr(p, 'shortcut'):
                        d['wsT'] = U.pack_linear_weight_dgrad(p.shortcut.weight, narrow=nw).to(dev)
                elif kind == 'attn':
                    d['wqkvT'] = U.pack_linear_weight_dgrad(p.qkv.weight, narrow=nw).to(dev)
                    d['wprojT'] = U.pack_linear_weight_dgrad(p.proj.weight, narrow=nw).to(dev)
                elif kind == 'down':
                    w = p.downsample.weight.detach().permute(0, 2, 3, 1).reshape(p.c, 9 * p.c)       # [c, tap*c + cin]
                    d['wT'] = U.pack_linear_weight_dgrad(w, narrow=nw).to(dev)
                elif kind == 'up':
                    d['wT'] = U.pack_conv_weight_dgrad(p.conv.weight, narrow=nw).to(dev)

        for seq, blk in zip(self.in_seq, list(m.in_blocks)[1:]):
            params(seq, blk)
        params(self.mid_seq, m.mid_blocks)
        for seq, blk in zip(self.out_seq, m.out_blocks):
            params(seq, blk)
        self.conv_in['wT'] = U.pack_conv_weight_dgrad(m.in_blocks[0][0].weight, narrow=nw).to(dev)      # K = base width, rows = cin
        self.out_conv['wT'] = U.pack_conv_weight_dgrad(m.out.conv.weight, cout_pad=self.CPAD_IN).to(dev)  # K = 18 -> 64, rows = 128
        self._bwd_packed = True

    GRAD_TARGET = 1024.0      # max |d loss / d v| after loss scaling: fp16 storage leaves 65504 / 1024 = 64x headroom inside the walk
    GRAD_RETRIES = 4          # walks after the first, each with the target divided by another 8 (down to 0.25: 262144x headroom)

    def backward_nchw(self, grad_v, weight_grads=False):
        """grad_v fp32 [B,C,H,W] (d loss / d v) -> d loss / d x_t fp32 [B,C,H,W], for the forward that just ran with save=True.
        weight_grads=True: the same walk also produces the parameter gradients (`unet_train.WeightGradPass`): returns
        (dx, grads, d_scale_shift).
        A finite grad_v whose gradients overflow the fp16 storage of the walk (d x_t comes out non-finite) is walked again from the same
        tape with the loss-scale target divided by 8, up to GRAD_RETRIES times; then the first layer that overflows is named in an error.
        A non-finite grad_v gives a non-finite result, as in fp32 autograd.  Costs one 8-byte device-to-host read per call."""
        from .unet_train import WeightGradPass
        B, C, H, W = grad_v.shape
        L, s = N.lib(), N.stream_ptr()
        scale = self._buf(('bwd', 'scale'), (4,), torch.float32)
        g_in = self._buf(('bwd', 'g_in'), (B, H, W, self.CPAD_IN))
        out = torch.empty(B, self.cin_total, H, W, dtype=torch.float32, device=self.dev)

        def walk(target, check=False):
            N.check(L.ssdnerf_grad_scale(N.ptr(grad_v), N.ctypes.c_ulonglong(grad_v.numel()), N.c_f32(target), N.ptr(scale), s))
            N.check(L.ssdnerf_grad_nchw_to_nhwc_f16(N.ptr(grad_v), N.c_u32(B), N.c_u32(C), N.c_u32(H), N.c_u32(W), N.c_u32(self.CPAD_IN),
                                                    N.ptr(scale), N.ptr(g_in), s))
            wg = WeightGradPass(self) if weight_grads else None       # fresh per walk: it accumulates
            dx = self.backward_nhwc(g_in, wg=wg, check=check)
            N.check(L.ssdnerf_grad_nhwc_to_nchw_f32(N.ptr(dx), N.c_u32(B), N.c_u32(self.cin_total), N.c_u32(H), N.c_u32(W),
                                                    N.c_u32(self.CPAD_IN), N.ptr(scale), N.ptr(out), s))
            return wg

        for k in range(self.GRAD_RETRIES + 1):
            target = self.GRAD_TARGET / 8 ** k
            wg = walk(target)
            grad_v_bad, dx_bad = scale[2:].tolist()
            if grad_v_bad or not dx_bad:
                break
        else:
            walk(target, check=True)          # raises naming the first layer whose gradient is not finite
            raise N.SSDNeRFNativeError(f'UNet backward: d x_t is not finite at loss-scale target {target} although d loss / d v is')
        if wg is not None:
            grads, d_ss = wg.finish(scale[1])
            return out, grads, d_ss
        return out

    def _layer_name(self, r):
        if r['kind'] == 'out':
            return 'out'
        if r['kind'] == 'conv_in':
            return 'in_blocks.0.0'
        return next(n for n, mod in self.m.named_modules() if mod is r['d']['mod'])

    def backward_nhwc(self, g_v, wg=None, check=False):
        """g_v fp16 [B,H,W,CPAD_IN] (loss-scaled d loss / d v, zero beyond the model's channels) -> fp32 [B,H,W,CPAD_IN] d loss / d x_in.
        Walks the tape of the last save=True forward in reverse; every convolution / linear gradient is the forward's tensor-core
        kernel on transposed weights, the rest are the section-4b glue kernels.  check=True (diagnosis, synchronises per layer): raise
        naming the first layer of the walk after which a gradient is not finite."""
        if not self.tape or self.tape[-1]['kind'] != 'out':
            raise N.SSDNeRFNativeError('UNet backward needs a preceding forward_nhwc(save=True)')
        if not self._bwd_packed:
            self._pack_backward_weights()
        L, s = N.lib(), N.stream_ptr
        nw, G = self.narrow, self.groups
        grads = {}

        def gb(name, idx, shape, dtype=torch.float16):
            return self._buf(('bwd', name, idx), shape, dtype)

        def acc(t, g):
            """gradient w.r.t. forward tensor t: first contribution is stored, later ones are added in place"""
            k = t.data_ptr()
            old = grads.get(k)
            if old is not None:
                N.check(L.ssdnerf_add_f16(N.ptr(g), N.ptr(old), N.ctypes.c_ulonglong(g.numel()), s()))
            grads[k] = g

        gsum = self._buf(('bwd', 'gsum'), (self.B * 64,), torch.float32)
        dx_in = None
        for idx in range(len(self.tape) - 1, -1, -1):
            r = self.tape[idx]
            kind = r['kind']
            if kind == 'out':
                x = r['x']
                B, H, W, c = x.shape
                d_a = U.conv3x3_f16(g_v, self.out_conv['wT'], c, out=gb('d_a', (H, c), (B, H, W, c)), narrow=nw)
                dh = gb('dx', idx, (B, H, W, c))
                cs = wg.csum(c) if wg else None
                U.gn_bwd(x, None, r['st'], self.out_norm['g'], self.out_norm['b'], d_a, dh, silu=True, gsum=gsum, csum=cs, groups=G)
                if wg:
                    wg.out(r, g_v, cs)
                acc(x, dh)
            elif kind == 'res':
                d, x, sk, h1, out = r['d'], r['x'], r['sk'], r['h1'], r['out']
                g = grads.pop(out.data_ptr())
                B, H, W, C1 = x.shape
                C2 = sk.shape[-1] if sk is not None else 0
                cin, cout = d['cin'], d['cout']
                d_a2 = U.conv3x3_f16(g, d['w2T'], cout, out=gb('d_a2', (H, cout), (B, H, W, cout)), narrow=nw)
                self._dropout(d_a2, d['idx'])                     # same mask as the forward (a no-op outside training)
                d_h1 = gb('d_h1', (H, cout), (B, H, W, cout))
                ss = N.c_void_p(self.ss_cur.data_ptr() + 4 * self.ss_offsets[d['idx']])
                cs2 = wg.csum(cout) if wg else None
                U.gn_bwd(h1, None, r['st2'], d['g2'], d['b2'], d_a2, d_h1, scale_shift_ptr=ss, ss_batch_stride=self.ss_total, silu=True, gsum=gsum,
                         csum=cs2, groups=G)
                if wg:      # conv_2 / norm 2 / embedding rows now: cs2 and the 'a' scratch are reused below
                    wg.res_second(r, g, cs2)
                d_a = U.conv3x3_f16(d_h1, d['w1T'], cin, out=gb('d_a', (H, cin), (B, H, W, cin)), narrow=nw)
                if 'wsT' in d:
                    add = U.conv3x3_f16(g, d['wsT'].unsqueeze(0), cin, taps=1, out=gb('d_sc', (H, cin), (B, H, W, cin)), narrow=nw)
                else:
                    assert sk is None and cin == cout
                    add = g
                dx = gb('dx', idx, (B, H, W, C1))
                dsk = gb('dsk', idx, (B, H, W, C2)) if sk is not None else None
                cs1 = wg.csum(cin) if wg else None
                U.gn_bwd(x, sk, r['st1'], d['g1'], d['b1'], d_a, dx, dsk, add=add, silu=True, gsum=gsum, csum=cs1, groups=G)
                if wg:
                    wg.res_first(r, g, d_h1, cs1)
                acc(x, dx)
                if sk is not None:
                    acc(sk, dsk)
            elif kind == 'attn':
                d, x, qkv, out = r['d'], r['x'], r['qkv'], r['out']
                g = grads.pop(out.data_ptr())
                B, H, W, c = x.shape
                T, heads = H * W, d['heads']
                d_o = U.linear_f16(g.view(B * T, c), d['wprojT'], n=c, out=gb('d_o', (T, c), (B * T, c)), narrow=nw)
                dqkv = U.attn_backward(qkv, d_o.view(B, T, c), heads, 1.0 / math.sqrt(c // heads),
                                       lambda name, shape, dtype: gb('att_' + name, (T, c), shape, dtype), narrow=nw)
                d_xn = U.linear_f16(dqkv.view(B * T, 3 * c), d['wqkvT'], n=c, out=gb('d_xn', (T, c), (B * T, c)), narrow=nw)
                dx = gb('dx', idx, (B, H, W, c))
                cs = wg.csum(c) if wg else None
                U.gn_bwd(x, None, r['st'], d['g'], d['b'], d_xn.view(B, H, W, c), dx, add=g, silu=False, gsum=gsum, csum=cs, groups=G)
                if wg:
                    wg.attn(r, g, dqkv, cs)
                acc(x, dx)
            elif kind == 'down':
                d, x, out = r['d'], r['x'], r['out']
                g = grads.pop(out.data_ptr())
                B, H, W, c = x.shape
                if wg:
                    wg.down(r, g)
                M = B * (H // 2) * (W // 2)
                dcol = U.linear_f16(g.view(M, c), d['wT'], n=9 * c, out=gb('dcol', (H, c), (M, 9 * c)), narrow=nw)
                dx = gb('dx', idx, (B, H, W, c))
                old = grads.pop(x.data_ptr(), None)
                N.check(L.ssdnerf_col2im_s2(N.ptr(dcol), N.c_u32(B), N.c_u32(H), N.c_u32(W), N.c_u32(c), N.ptr(old), N.ptr(dx), s()))
                grads[x.data_ptr()] = dx
            elif kind == 'up':
                d, x, out = r['d'], r['x'], r['out']
                g = grads.pop(out.data_ptr())
                B, H, W, c = x.shape
                if wg:
                    wg.up(r, g)
                dup = U.conv3x3_f16(g, d['wT'], c, out=gb('dup', (H, c), (B, 2 * H, 2 * W, c)), narrow=nw)
                dx = gb('dx', idx, (B, H, W, c))
                N.check(L.ssdnerf_sum2x2(N.ptr(dup), N.c_u32(B), N.c_u32(H), N.c_u32(W), N.c_u32(c), N.ptr(dx), s()))
                acc(x, dx)
            elif kind == 'conv_in':
                g = grads.pop(r['out'].data_ptr())
                if wg:
                    wg.conv_in(r, g)
                dx_in = self._buf(('bwd', 'dx_in'), (self.B, self.H, self.W, self.CPAD_IN), torch.float32)
                U.conv3x3_f16(g, self.conv_in['wT'], self.cin_total, out=dx_in, narrow=nw)
            if check and not all(bool(torch.isfinite(t).all()) for t in list(grads.values()) + ([dx_in] if dx_in is not None else [])):
                raise N.SSDNeRFNativeError(f'UNet backward: the fp16 gradients overflow at layer `{self._layer_name(r)}` even with the '
                                           f'loss scale lowered {8 ** self.GRAD_RETRIES}x (forward activations or weights out of range?)')
        assert not grads, 'dangling gradients in the UNet tape'
        return dx_in

    def load_input_nchw(self, x):
        """x fp32 [B,C,H,W] -> self.x_in"""
        B, C, H, W = x.shape
        N.check(N.lib().ssdnerf_nchw_to_nhwc_f16(N.ptr(x), N.c_u32(B), N.c_u32(C), N.c_u32(H), N.c_u32(W), N.c_u32(self.CPAD_IN),
                                                 N.ptr(self.x_in), N.stream_ptr()))

    def forward_nchw(self, x):
        self.load_input_nchw(x)
        return self.forward_nhwc()
