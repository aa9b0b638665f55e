"""FPN / ResNet backbone plugin on libmdt_b200 convs — same constructor, attribute names and output list as the reference's
models/backbone.py:22-218 (`FPN(cf, conv, operate_stride1=False)`, `forward(x) -> [P0?, P2, P3, P4, P5, (P6)]`), so it can be named in
`cf.backbone_path` (mrcnn.py:842-847, retina_unet.py:370-375) and loads the reference's state dicts key-for-key.

H100 specifics: activations stay NDHWC (channels_last_3d) end to end; bias/ReLU run in the conv epilogues; the residual add + ReLU of a
bottleneck block is fused into the epilogue of its third conv (backbone.py:195-206 does conv3 -> += residual -> ReLU as three passes).
"""
import torch
import torch.nn as nn
import torch.nn.functional as F

try:
    from . import _lib as L
    from .conv import Conv3d, Conv2d, _Conv3dFn, no_split_consumer, pointwise_eligible
    from .norm import LeakyReLU
except ImportError:   # loaded by FILE PATH as the reference does (utils.import_module('bbone', cf.backbone_path), mrcnn.py:842): no parent package
    from medicaldetectiontoolkit_b200 import _lib as L
    from medicaldetectiontoolkit_b200.conv import Conv3d, Conv2d, _Conv3dFn, no_split_consumer, pointwise_eligible
    from medicaldetectiontoolkit_b200.norm import LeakyReLU

_CL3 = torch.channels_last_3d


def _to_cl(x):
    return x.contiguous(memory_format=_CL3) if x.dim() == 5 else x.contiguous(memory_format=torch.channels_last)


def _fused_residual_relu(conv_mod, x, residual, relu=True):
    """relu?(conv(x) + bias + residual) in one kernel when conv_mod is a bare libmdt conv; generic fallback otherwise"""
    if isinstance(conv_mod, Conv3d):
        return _Conv3dFn.apply(x, conv_mod.weight, conv_mod.bias, _to_cl(residual), conv_mod.stride, conv_mod.padding, relu, conv_mod.precision,
                               conv_mod.algo, conv_mod.emit_split)
    if isinstance(conv_mod, Conv2d):
        y = _Conv3dFn.apply(x.unsqueeze(2), conv_mod.weight.unsqueeze(2), conv_mod.bias, residual.unsqueeze(2), (1,) + conv_mod.stride,
                            (0,) + conv_mod.padding, relu, conv_mod.precision, conv_mod.algo)
        return y.squeeze(2)
    return None


class ResBlock(nn.Module):
    """bottleneck block: 1x1 (stride) -> 3x3 -> 1x1 (x4) + shortcut -> ReLU   (models/backbone.py:183-206)"""

    def __init__(self, start_filts, planes, conv, stride=1, downsample=None, norm=None, relu='relu'):
        super().__init__()
        self.conv1 = conv(start_filts, planes, ks=1, stride=stride, norm=norm, relu=relu)
        self.conv2 = conv(planes, planes, ks=3, pad=1, norm=norm, relu=relu)
        self.conv3 = conv(planes, planes * 4, ks=1, norm=norm, relu=None)
        self.relu = nn.ReLU(inplace=True) if relu == 'relu' else LeakyReLU(inplace=True)
        self.downsample = None
        if downsample is not None:
            self.downsample = conv(downsample[0], downsample[0] * downsample[1], ks=1, stride=downsample[2], norm=norm, relu=None)
        self.stride = stride
        self._fusable = (relu == 'relu') and norm is None
        # with a norm, conv3 is Sequential(conv, norm) and the add + activation run in the norm's apply pass
        self._act = relu if norm is not None else None
        # split planes are emitted for tensor-core consumers only: conv3 (1x1x1) reads fp32 rows when it is pointwise-eligible, and the block
        # output mostly feeds the next block's 1x1x1 conv1 / a lateral (the few strided or wide consumers split on demand)
        if pointwise_eligible(planes, planes * 4):
            no_split_consumer(self.conv2)
        no_split_consumer(self.conv3)

    def forward(self, x):
        shortcut = self.downsample(x) if self.downsample is not None else x
        out = self.conv2(self.conv1(x))
        if self._fusable:
            fused = _fused_residual_relu(self.conv3, out, shortcut)
            if fused is not None:
                return fused
        elif self._act is not None:
            return self.conv3[1].norm_act(self.conv3[0](out), residual=shortcut, act=self._act)
        elif isinstance(self.relu, LeakyReLU):
            fused = _fused_residual_relu(self.conv3, out, shortcut, relu=False)
            if fused is not None:
                return self.relu(fused)
        return self.relu(self.conv3(out) + shortcut)


class _Upsample221(torch.autograd.Function):
    """(2,2,1) trilinear up-sampling of a channels-last map on libmdt_b200 (csrc/resample.cu); backward = gather adjoint.  any_c selects
    mdt_upsample_linear2x_* (any channel count, V = 4 / 2 / 1 channels per access) instead of the float4-only mdt_upsample221_*"""

    @staticmethod
    def forward(ctx, x, any_c=False):
        lib = L.load()
        x = _cl3_aligned(x)
        n, c, d, h, w = x.shape
        y = torch.empty((n, c, 2 * d, 2 * h, w), dtype=x.dtype, device=x.device, memory_format=_CL3)
        fwd = lib.mdt_upsample_linear2x_forward if any_c else lib.mdt_upsample221_forward
        with torch.cuda.device(x.device):
            L.check(fwd(L.ptr(x), L.ptr(y), n, d, h, w, c, L.stream_ptr()))
        ctx.shape = (n, c, d, h, w)
        ctx.any_c = any_c
        return y

    @staticmethod
    def backward(ctx, gy):
        lib = L.load()
        n, c, d, h, w = ctx.shape
        gy = _cl3_aligned(gy)
        gx = torch.empty((n, c, d, h, w), dtype=gy.dtype, device=gy.device, memory_format=_CL3)
        bwd = lib.mdt_upsample_linear2x_backward if ctx.any_c else lib.mdt_upsample221_backward
        with torch.cuda.device(gy.device):
            L.check(bwd(L.ptr(gy), L.ptr(gx), n, d, h, w, c, L.stream_ptr()))
        return gx, None


def _cl3_aligned(t):
    """t as a channels-last-3d tensor whose data pointer is 16-byte aligned: .contiguous() keeps the storage offset of an already-contiguous
    view, and the float4 paths of csrc/resample.cu refuse a misaligned base (MDT_EINVAL) while the others fall back to narrower accesses, so
    such a view is copied"""
    t = t.contiguous(memory_format=_CL3)
    return t if t.data_ptr() % 16 == 0 else t.clone(memory_format=_CL3)


def _i3(vals):
    import ctypes
    return (ctypes.c_int * 3)(*[int(v) for v in vals])


class _MaxPoolFn(torch.autograd.Function):
    """channels-last max pooling on libmdt_b200 (csrc/resample.cu): forward keeps one arg-max byte per element, backward is a gather"""

    @staticmethod
    def forward(ctx, x, kernel, stride, pad):
        lib = L.load()
        x = _cl3_aligned(x)
        n, c, d, h, w = x.shape
        od, oh, ow = [(i + 2 * p - k) // s + 1 for i, k, s, p in zip((d, h, w), kernel, stride, pad)]
        y = torch.empty((n, c, od, oh, ow), dtype=x.dtype, device=x.device, memory_format=_CL3)
        arg = torch.empty((n, od, oh, ow, c), dtype=torch.uint8, device=x.device)
        with torch.cuda.device(x.device):
            L.check(lib.mdt_maxpool3d_forward(L.ptr(x), L.ptr(y), L.ptr(arg), n, d, h, w, c, _i3(kernel), _i3(stride), _i3(pad), L.stream_ptr()))
        ctx.save_for_backward(arg)
        ctx.geom = (n, c, d, h, w, kernel, stride, pad)
        return y

    @staticmethod
    def backward(ctx, gy):
        lib = L.load()
        (arg,) = ctx.saved_tensors
        n, c, d, h, w, kernel, stride, pad = ctx.geom
        gy = _cl3_aligned(gy)
        gx = torch.empty((n, c, d, h, w), dtype=gy.dtype, device=gy.device, memory_format=_CL3)
        with torch.cuda.device(gy.device):
            L.check(lib.mdt_maxpool3d_backward(L.ptr(gy), L.ptr(arg), L.ptr(gx), n, d, h, w, c, _i3(kernel), _i3(stride), _i3(pad), L.stream_ptr()))
        return gx, None, None, None


class MaxPool(nn.Module):
    """nn.MaxPool3d(kernel_size=3, stride=(2,2,1), padding=1) / nn.MaxPool2d(3, 2, 1) in front of C2 (models/backbone.py:63-64) on the library's
    own kernels for CUDA fp32 maps; parameter-free, so the state-dict keys of `C2` are unchanged"""

    def __init__(self, dim, kernel_size, stride, padding):
        super().__init__()
        t = lambda v: tuple(v) if isinstance(v, (tuple, list)) else (v,) * dim
        self.dim = dim
        self.kernel_size, self.stride, self.padding = t(kernel_size), t(stride), t(padding)

    def forward(self, x):
        if not (x.is_cuda and x.dtype == torch.float32):
            pool = F.max_pool3d if self.dim == 3 else F.max_pool2d
            return pool(x, self.kernel_size, self.stride, self.padding)
        if self.dim == 3:
            return _MaxPoolFn.apply(x, self.kernel_size, self.stride, self.padding)
        y = _MaxPoolFn.apply(x.unsqueeze(2), (1,) + self.kernel_size, (1,) + self.stride, (0,) + self.padding)
        return y.squeeze(2)


class _NearestUp2Fn(torch.autograd.Function):
    """F.interpolate(x, scale_factor=2) (nearest) of the FPN top-down path (models/backbone.py:147-153) on csrc/resample.cu; backward = child sum"""

    @staticmethod
    def forward(ctx, x, fd):
        lib = L.load()
        x = _cl3_aligned(x)
        n, c, d, h, w = x.shape
        y = torch.empty((n, c, d * fd, 2 * h, 2 * w), dtype=x.dtype, device=x.device, memory_format=_CL3)
        with torch.cuda.device(x.device):
            L.check(lib.mdt_upsample_nearest_forward(L.ptr(x), L.ptr(y), n, d, h, w, c, fd, 2, 2, L.stream_ptr()))
        ctx.geom = (n, c, d, h, w, fd)
        return y

    @staticmethod
    def backward(ctx, gy):
        lib = L.load()
        n, c, d, h, w, fd = ctx.geom
        gy = _cl3_aligned(gy)
        gx = torch.empty((n, c, d, h, w), dtype=gy.dtype, device=gy.device, memory_format=_CL3)
        with torch.cuda.device(gy.device):
            L.check(lib.mdt_upsample_nearest_backward(L.ptr(gy), L.ptr(gx), n, d, h, w, c, fd, 2, 2, L.stream_ptr()))
        return gx, None


def nearest_up2(x):
    """nearest x2 along every spatial axis, own kernels for CUDA fp32 maps (5-D: all three axes, 4-D: both)"""
    if not (x.is_cuda and x.dtype == torch.float32):
        return F.interpolate(x, scale_factor=2)
    if x.dim() == 5:
        return _NearestUp2Fn.apply(x, 2)
    return _NearestUp2Fn.apply(x.unsqueeze(2), 1).squeeze(2)


class Interpolate(nn.Module):
    def __init__(self, scale_factor, mode):
        super().__init__()
        self.scale_factor = scale_factor
        self.mode = mode

    def forward(self, x):
        """CUDA fp32 maps run on the library: 5-D trilinear (2,2,1) (float4 kernels at C % 4 == 0, any C otherwise) and 4-D bilinear x2 as
        the same map of x.unsqueeze(-1) (channels-last-3d with w = 1); both backwards are fixed-order gathers"""
        if x.is_cuda and x.dtype == torch.float32:
            sf = tuple(self.scale_factor) if isinstance(self.scale_factor, (tuple, list)) else (self.scale_factor,) * (x.dim() - 2)
            if x.dim() == 5 and self.mode == 'trilinear' and sf == (2, 2, 1):
                return _Upsample221.apply(x, x.shape[1] % 4 != 0)
            if x.dim() == 4 and self.mode == 'bilinear' and sf == (2, 2):
                return _Upsample221.apply(x.unsqueeze(-1), True).squeeze(-1)
        return F.interpolate(x, scale_factor=self.scale_factor, mode=self.mode, align_corners=False)


class FPN(nn.Module):
    """Feature pyramid over a ResNet-50/101-style encoder; optional full-resolution decoder levels P1/P0 (`operate_stride1`)."""

    def __init__(self, cf, conv, operate_stride1=False):
        super().__init__()
        sf = cf.start_filts
        self.start_filts = sf
        self.n_blocks = [3, 4, {"resnet50": 6, "resnet101": 23}[cf.res_architecture], 3]
        self.block = ResBlock
        self.block_expansion = 4
        self.operate_stride1 = operate_stride1
        self.sixth_pooling = cf.sixth_pooling
        self.dim = conv.dim
        three_d = conv.dim == 3
        s221 = (2, 2, 1) if three_d else 2
        blk = dict(conv=conv, norm=cf.norm, relu=cf.relu)

        if operate_stride1:
            self.C0 = nn.Sequential(conv(cf.n_channels, sf, ks=3, pad=1, norm=cf.norm, relu=cf.relu),
                                    conv(sf, sf, ks=3, pad=1, norm=cf.norm, relu=cf.relu))
            self.C1 = conv(sf, sf, ks=7, stride=s221, pad=3, norm=cf.norm, relu=cf.relu)
        else:
            self.C1 = conv(cf.n_channels, sf, ks=7, stride=s221, pad=3, norm=cf.norm, relu=cf.relu)

        sfe = sf * self.block_expansion

        def stage(c_in, planes, n, stride, first_downsample):
            layers = [ResBlock(c_in, planes, stride=stride, downsample=first_downsample, **blk)]
            layers += [ResBlock(planes * 4, planes, **blk) for _ in range(1, n)]
            return layers

        pool = MaxPool(3, 3, (2, 2, 1), 1) if three_d else MaxPool(2, 3, 2, 1)
        self.C2 = nn.Sequential(pool, *stage(sf, sf, self.n_blocks[0], 1, (sf, self.block_expansion, 1)))
        self.C3 = nn.Sequential(*stage(sfe, sf * 2, self.n_blocks[1], 2, (sfe, 2, 2)))
        self.C4 = nn.Sequential(*stage(sfe * 2, sf * 4, self.n_blocks[2], 2, (sfe * 2, 2, 2)))
        self.C5 = nn.Sequential(*stage(sfe * 4, sf * 8, self.n_blocks[3], 2, (sfe * 4, 2, 2)))
        if self.sixth_pooling:
            self.C6 = nn.Sequential(*stage(sfe * 8, sf * 16, self.n_blocks[3], 2, (sfe * 8, 2, 2)))

        up = dict(scale_factor=(2, 2, 1), mode='trilinear') if three_d else dict(scale_factor=2, mode='bilinear')
        self.P1_upsample = Interpolate(**up)
        self.P2_upsample = Interpolate(**up)

        oc = cf.end_filts
        self.out_channels = oc
        self.P5_conv1 = conv(sf * 32 + cf.n_latent_dims, oc, ks=1, stride=1, relu=None)
        self.P4_conv1 = conv(sf * 16, oc, ks=1, stride=1, relu=None)
        self.P3_conv1 = conv(sf * 8, oc, ks=1, stride=1, relu=None)
        self.P2_conv1 = conv(sf * 4, oc, ks=1, stride=1, relu=None)
        self.P1_conv1 = no_split_consumer(conv(sf, oc, ks=1, stride=1, relu=None))   # p1_pre only feeds the (2,2,1) up-sampling
        if operate_stride1:
            self.P0_conv1 = conv(sf, oc, ks=1, stride=1, relu=None)
            self.P0_conv2 = conv(oc, oc, ks=3, stride=1, pad=1, relu=None)
        self.P1_conv2 = conv(oc, oc, ks=3, stride=1, pad=1, relu=None)
        self.P2_conv2 = conv(oc, oc, ks=3, stride=1, pad=1, relu=None)
        self.P3_conv2 = conv(oc, oc, ks=3, stride=1, pad=1, relu=None)
        self.P4_conv2 = conv(oc, oc, ks=3, stride=1, pad=1, relu=None)
        self.P5_conv2 = conv(oc, oc, ks=3, stride=1, pad=1, relu=None)
        if self.sixth_pooling:
            self.P6_conv1 = conv(sf * 64, oc, ks=1, stride=1, relu=None)
            self.P6_conv2 = conv(oc, oc, ks=3, stride=1, pad=1, relu=None)

    @staticmethod
    def _conv_plus(conv_mod, c, other):
        """conv(c) + other with the add fused into the conv epilogue when conv_mod is a bare libmdt conv"""
        if isinstance(conv_mod, Conv3d):
            return _Conv3dFn.apply(c, conv_mod.weight, conv_mod.bias, _to_cl(other), conv_mod.stride, conv_mod.padding, False, conv_mod.precision,
                                   conv_mod.algo, conv_mod.emit_split)
        return conv_mod(c) + other

    @staticmethod
    def _lateral(conv_mod, c, top):
        """lateral 1x1 conv + nearest x2 upsampled coarser map, the add fused into the conv epilogue when possible"""
        up = nearest_up2(top)
        fused = None
        if isinstance(conv_mod, Conv3d):
            fused = _Conv3dFn.apply(c, conv_mod.weight, conv_mod.bias, _to_cl(up), conv_mod.stride, conv_mod.padding, False, conv_mod.precision,
                                    conv_mod.algo, conv_mod.emit_split)
        return fused if fused is not None else conv_mod(c) + up

    def forward(self, x):
        """x [b, c, y, x, (z)] -> list of pyramid maps, finest first: [P0 (if operate_stride1), P2, P3, P4, P5, (P6)]"""
        x = _to_cl(x)
        c0 = self.C0(x) if self.operate_stride1 else x
        c1 = self.C1(c0)
        c2 = self.C2(c1)
        c3 = self.C3(c2)
        c4 = self.C4(c3)
        c5 = self.C5(c4)
        if self.sixth_pooling:
            c6 = self.C6(c5)
            p6_pre = self.P6_conv1(c6)
            p5_pre = self._lateral(self.P5_conv1, c5, p6_pre)
        else:
            p5_pre = self.P5_conv1(c5)
        p4_pre = self._lateral(self.P4_conv1, c4, p5_pre)
        p3_pre = self._lateral(self.P3_conv1, c3, p4_pre)
        p2_pre = self._lateral(self.P2_conv1, c2, p3_pre)

        outs = [self.P2_conv2(p2_pre), self.P3_conv2(p3_pre), self.P4_conv2(p4_pre), self.P5_conv2(p5_pre)]
        if self.sixth_pooling:
            outs.append(self.P6_conv2(p6_pre))
        if self.operate_stride1:
            p1_pre = self._conv_plus(self.P1_conv1, c1, self.P2_upsample(p2_pre))
            p0_pre = self._conv_plus(self.P0_conv1, c0, self.P1_upsample(p1_pre))
            # P1_conv2 exists (and is in the state dict) but is unused, as in the reference (backbone.py:175)
            outs = [self.P0_conv2(p0_pre)] + outs
        return outs
