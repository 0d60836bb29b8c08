"""`spconv.pytorch`-compatible module surface on the virconv_b200 kernels — the drop-in boundary.

Mirrors what the reference imports through `pcdet/utils/spconv_utils.py:33-36` and uses in
`pcdet/models/backbones_3d/spconv_backbone.py`, `backbones_2d/map_to_bev/height_compression.py:29` and
`roi_heads/ted_head.py:507-541`:
    SparseConvTensor(features, indices, spatial_shape, batch_size)  .features .indices .spatial_shape
        .batch_size .indice_dict .dense() .replace_feature()
    SubMConv3d / SubMConv2d / SparseConv3d / SparseConv2d(in, out, kernel, stride, padding, dilation,
        groups, bias, indice_key)   parameter `weight` of shape (C_out, *kernel, C_in) (spconv 2.x layout,
        detector3d_template.py:358-370), leaf modules (optimizer flattening, optimization/__init__.py:26-27)
    SparseSequential, SparseModule, conv.SparseConvolution (spconv_utils.py:49)
`install_as_spconv()` registers these under the names `spconv`, `spconv.pytorch`, `spconv.pytorch.conv` so
the reference's own files import them unchanged.

Everything runs on CUDA tensors through the C ABI; a CPU tensor raises.
"""
from __future__ import annotations

import math
import sys
import types

import numpy as np
import torch
import torch.nn as nn

from . import ops


class SparseConvTensor:
    def __init__(self, features, indices, spatial_shape, batch_size, grid=None, voxel_num=None, indice_dict=None,
                 benchmark=False):
        self._features = features
        self.indices = indices               # assignable, spconv_backbone.py:147
        self.spatial_shape = list(spatial_shape)
        self.batch_size = batch_size
        self.indice_dict = indice_dict if indice_dict is not None else {}
        self.grid = grid
        self.voxel_num = voxel_num
        self.benchmark = benchmark
        self._features_bf16 = None           # optional bf16 shadow of `features` (tensor-core operand), see ops.py
        self.num_rows = None                 # static (graph) mode only: device row count of capacity-sized features / indices

    @property
    def features_bf16(self):
        v = self._features_bf16
        if callable(v):                      # plan-executor tensors resolve their shadow on first use
            v = self._features_bf16 = v()
        return v

    @features_bf16.setter
    def features_bf16(self, val):
        self._features_bf16 = val

    @property
    def features(self):
        return self._features

    @features.setter
    def features(self, val):
        raise ValueError("you can't set feature directly, use 'x = x.replace_feature(your_new_feature)' "
                         "to generate new SparseConvTensor instead.")

    def replace_feature(self, feature):
        return SparseConvTensor(feature, self.indices, self.spatial_shape, self.batch_size, self.grid, self.voxel_num,
                                self.indice_dict, self.benchmark)

    @property
    def spatial_size(self):
        return int(torch.tensor(self.spatial_shape).prod())

    def find_indice_pair(self, key):
        return None if key is None else self.indice_dict.get(key)

    def dense(self, channels_first=True):
        if self.num_rows is None:
            out = ops.DenseFn.apply(self._features, _as_i32(self.indices), self.batch_size, self.spatial_shape)
        else:           # static mode: only the valid rows are scattered (the index tail is -1)
            out = ops.DenseFn.apply(self._features, _as_i32(self.indices), self.batch_size, self.spatial_shape, self.num_rows)
        if channels_first:
            return out
        nd = len(self.spatial_shape)
        return out.permute(0, *range(2, nd + 2), 1).contiguous()


def _as_i32(indices):
    if indices.dtype != torch.int32 or not indices.is_contiguous():
        indices = indices.to(torch.int32).contiguous()
    return indices


class SparseModule(nn.Module):
    """Marker base class: modules that take and return a SparseConvTensor."""
    pass


class SparseConvolution(SparseModule):
    def __init__(self, ndim, in_channels, out_channels, kernel_size=3, stride=1, padding=0, dilation=1, groups=1,
                 bias=True, subm=False, output_padding=0, transposed=False, inverse=False, indice_key=None,
                 algo=None, fp32_accum=None, name=None):
        super().__init__()
        if groups != 1:
            raise NotImplementedError('groups != 1 is not used by VirConv and not implemented')
        if transposed or inverse:
            raise NotImplementedError('inverse / transposed sparse conv is not on the VirConv path '
                                      '(post_act_block conv_type="inverseconv" is never selected)')
        tup = lambda v: tuple(v) if isinstance(v, (list, tuple)) else (v,) * ndim
        self.ndim = ndim
        self.in_channels, self.out_channels = in_channels, out_channels
        self.kernel_size, self.stride = tup(kernel_size), tup(stride)
        self.padding, self.dilation = tup(padding), tup(dilation)
        self.conv1x1 = all(k == 1 for k in self.kernel_size)
        if subm and any(k % 2 == 0 for k in self.kernel_size):
            # (spconv asserts the same; the dgrad of a submanifold conv reuses the forward table with mirrored offsets,
            #  which is only its own transpose for odd, symmetric kernels)
            raise ValueError(f'submanifold convolution needs odd kernel sizes, got {self.kernel_size}')
        self.subm, self.indice_key = subm, indice_key
        self.groups = groups
        self.precision = 'fp32'      # 'bf16' -> wgmma tensor-core kernels (see ops.py); set via set_precision()
        self.weight = nn.Parameter(torch.empty(out_channels, *self.kernel_size, in_channels))
        if bias:
            self.bias = nn.Parameter(torch.empty(out_channels))
        else:
            self.register_parameter('bias', None)
        self.reset_parameters()

    def reset_parameters(self):
        nn.init.kaiming_uniform_(self.weight, a=math.sqrt(5))
        if self.bias is not None:
            fan_in = self.in_channels * int(torch.tensor(self.kernel_size).prod())
            bound = 1 / math.sqrt(fan_in)
            nn.init.uniform_(self.bias, -bound, bound)

    def extra_repr(self):
        return (f'{self.in_channels}, {self.out_channels}, kernel_size={self.kernel_size}, stride={self.stride}, '
                f'padding={self.padding}, subm={self.subm}, indice_key={self.indice_key}')

    # -- rulebook (cached in the tensor's indice_dict under indice_key, as spconv does) ---------------
    def rulebook(self, x: SparseConvTensor) -> ops.Rulebook:
        key = self.indice_key
        indices = _as_i32(x.indices)
        cached = x.indice_dict.get(key) if key is not None else None
        if cached is not None and isinstance(cached, ops.Rulebook):
            if self.subm and cached.n_in != indices.shape[0]:
                raise ValueError(f'indice_key {key!r} was built for {cached.n_in} rows, tensor has {indices.shape[0]}')
            return cached
        # VirConv gives every layer its own indice_key (spconv_backbone.py:170-205) although d3_conv1/d3_conv2
        # (and d2_conv1/d2_conv2) see identical indices: reuse by geometry + identity of the index tensor.
        geo = ('__geo__', self.subm, self.ndim, self.kernel_size, self.stride, self.padding, self.dilation,
               indices.data_ptr(), indices.shape[0], indices._version, tuple(x.spatial_shape))
        rb = x.indice_dict.get(geo)
        if rb is None:
            if self.subm:
                rb = ops.build_subm_rulebook(indices, x.batch_size, x.spatial_shape, self.kernel_size, self.dilation)
            else:
                rb = ops.build_conv_rulebook(indices, x.batch_size, x.spatial_shape, self.kernel_size, self.stride,
                                             self.padding, self.dilation)
            rb._keepalive = indices
            x.indice_dict[geo] = rb
        if key is not None:
            x.indice_dict[key] = rb
        return rb

    def _out_tensor(self, x, feats, rb):
        if self.subm:
            return SparseConvTensor(feats, x.indices, x.spatial_shape, x.batch_size, x.grid, x.voxel_num, x.indice_dict,
                                    x.benchmark)
        return SparseConvTensor(feats, rb.out_indices, rb.out_shape, x.batch_size, x.grid, x.voxel_num, x.indice_dict,
                                x.benchmark)

    def forward(self, x: SparseConvTensor):
        assert isinstance(x, SparseConvTensor)
        rb = self.rulebook(x)
        out = ops.SparseConvFn.apply(x.features, self.weight, rb, self.precision)
        if self.bias is not None:
            out = out + self.bias
        return self._out_tensor(x, out, rb)

    def forward_bn_relu(self, x: SparseConvTensor, bn: nn.BatchNorm1d):
        """conv + BatchNorm1d + ReLU in one autograd node (the SparseSequential fast path)."""
        rb = self.rulebook(x)
        training = bn.training or (bn.running_mean is None)
        if bn.momentum is None:
            raise ValueError('cumulative-average BatchNorm (momentum=None) is not fused; SparseSequential routes it through torch')
        momentum = bn.momentum
        res = ops.ConvBNReLUFn.apply(x.features, self.weight, bn.weight, bn.bias, bn.running_mean, bn.running_var, rb,
                                     training, bn.eps, momentum, self.precision, x.features_bf16, bn.num_batches_tracked)
        if isinstance(res, tuple):
            out = self._out_tensor(x, res[0], rb)
            out.features_bf16 = res[1]
            return out
        return self._out_tensor(x, res, rb)


def set_precision(module: nn.Module, precision: str):
    """Select 'fp32' (parity) or 'bf16' (tensor-core) kernels for every sparse conv under `module`."""
    assert precision in ('fp32', 'bf16')
    for m in module.modules():
        if isinstance(m, SparseConvolution):
            m.precision = precision
    return module


def _make(ndim, subm):
    def __init__(self, in_channels, out_channels, kernel_size, stride=1, padding=0, dilation=1, groups=1, bias=True,
                 indice_key=None, algo=None, fp32_accum=None, name=None):
        SparseConvolution.__init__(self, ndim, in_channels, out_channels, kernel_size, stride, padding, dilation, groups,
                                   bias, subm, indice_key=indice_key)
    return __init__


class SubMConv3d(SparseConvolution):
    __init__ = _make(3, True)


class SubMConv2d(SparseConvolution):
    __init__ = _make(2, True)


class SparseConv3d(SparseConvolution):
    __init__ = _make(3, False)


class SparseConv2d(SparseConvolution):
    __init__ = _make(2, False)


class SparseInverseConv3d(SparseConvolution):
    def __init__(self, *a, **k):
        raise NotImplementedError('SparseInverseConv3d is not on the VirConv path')


class SparseInverseConv2d(SparseConvolution):
    def __init__(self, *a, **k):
        raise NotImplementedError('SparseInverseConv2d is not on the VirConv path')


class SparseSequential(SparseModule):
    """Applies sparse modules to the tensor and dense modules to `.features` (spconv semantics); the
    [conv(bias=False), BatchNorm1d, ReLU] triple every VirConv layer uses is dispatched as one fused op."""

    def __init__(self, *args, **kwargs):
        super().__init__()
        if len(args) == 1 and isinstance(args[0], dict):
            for k, m in args[0].items():
                self.add_module(k, m)
        else:
            for i, m in enumerate(args):
                self.add_module(str(i), m)
        for k, m in kwargs.items():
            self.add_module(k, m)

    def __getitem__(self, idx):
        return list(self._modules.values())[idx]

    def __len__(self):
        return len(self._modules)

    def add(self, module, name=None):
        self.add_module(name if name is not None else str(len(self._modules)), module)

    def forward(self, x):
        mods = list(self._modules.values())
        i = 0
        while i < len(mods):
            m = mods[i]
            if (isinstance(m, SparseConvolution) and m.bias is None and i + 2 < len(mods)
                    and type(mods[i + 1]) is nn.BatchNorm1d and mods[i + 1].affine and mods[i + 1].momentum is not None
                    and mods[i + 1].track_running_stats and isinstance(mods[i + 2], nn.ReLU)
                    and isinstance(x, SparseConvTensor) and x.indices.shape[0] > 0):
                x = m.forward_bn_relu(x, mods[i + 1])
                i += 3
                continue
            if isinstance(m, SparseModule):
                x = m(x)
            elif isinstance(x, SparseConvTensor):
                if x.indices.shape[0] != 0:
                    x = x.replace_feature(m(x.features))
            else:
                x = m(x)
            i += 1
        return x


# namespace objects ------------------------------------------------------------------------------------
conv = types.ModuleType(__name__ + '.conv')
conv.SparseConvolution = SparseConvolution
conv.SubMConv3d, conv.SubMConv2d = SubMConv3d, SubMConv2d
conv.SparseConv3d, conv.SparseConv2d = SparseConv3d, SparseConv2d


class _TVArray:
    """Stand-in for a `cumm.tensorview` array on the dataloader path: the reference only wraps numpy arrays on the way
    in (`tv.from_numpy`, data_processor.py:53) and calls `.numpy()` on the way out (:56-58)."""

    def __init__(self, arr):
        self._a = arr

    def numpy(self):
        return np.array(self._a, copy=True)       # "make copy with numpy()" (data_processor.py:55)

    def numpy_view(self):
        return self._a

    @property
    def shape(self):
        return list(self._a.shape)


class Point2VoxelCPU3d:
    """`spconv.utils.Point2VoxelCPU3d` as the reference's dataloader uses it (data_processor.py:24,35-41,53-58): first-come
    voxelisation on the host, coordinates emitted zyx.  The GPU path of this repo voxelises inside the model
    (preprocess.PointsToVoxels -> vc_voxelize_mean); this class only keeps `tools/train.py`'s unmodified dataset code
    importable and produces the same arrays (voxel order = first appearance, <= max_num_points_per_voxel points in point
    order, zero padded) through scenes.voxelize_first_come."""

    def __init__(self, vsize_xyz, coors_range_xyz, num_point_features, max_num_points_per_voxel, max_num_voxels):
        self.vsize_xyz = [float(v) for v in vsize_xyz]
        self.coors_range_xyz = [float(v) for v in coors_range_xyz]
        self.num_point_features = int(num_point_features)
        self.max_num_points_per_voxel = int(max_num_points_per_voxel)
        self.max_num_voxels = int(max_num_voxels)
        rng = np.asarray(self.coors_range_xyz, dtype=np.float64)
        self.grid_size = np.round((rng[3:] - rng[:3]) / np.asarray(self.vsize_xyz, dtype=np.float64)).astype(np.int64).tolist()

    def point_to_voxel(self, pc):
        from . import scenes
        pts = pc.numpy_view() if isinstance(pc, _TVArray) else np.asarray(pc)
        assert pts.ndim == 2 and pts.shape[1] == self.num_point_features, (pts.shape, self.num_point_features)
        voxels, coords, num = scenes.voxelize_first_come(pts, self.vsize_xyz, self.coors_range_xyz,
                                                         self.max_num_points_per_voxel, self.max_num_voxels)
        return _TVArray(voxels), _TVArray(coords), _TVArray(num)


def install_as_spconv():
    """Make `import spconv.pytorch as spconv` (pcdet/utils/spconv_utils.py:33-36), `from spconv.utils import
    Point2VoxelCPU3d` (data_processor.py:24) and `import cumm.tensorview as tv` (data_processor.py:10) resolve to this
    module's implementations.  `cumm` is only registered when no real one is importable."""
    me = sys.modules[__name__]
    pkg = types.ModuleType('spconv')
    pkg.__path__ = []
    pkg.pytorch = me
    pkg.__version__ = '2.1.22+virconv_b200'
    utils = types.ModuleType('spconv.utils')
    utils.Point2VoxelCPU3d = Point2VoxelCPU3d
    pkg.utils = utils
    sys.modules['spconv'] = pkg
    sys.modules['spconv.pytorch'] = me
    sys.modules['spconv.pytorch.conv'] = conv
    sys.modules['spconv.utils'] = utils
    if 'cumm' not in sys.modules:
        try:
            import cumm.tensorview  # noqa: F401
        except Exception:           # noqa: BLE001
            cumm = types.ModuleType('cumm')
            cumm.__path__ = []
            tvm = types.ModuleType('cumm.tensorview')
            tvm.from_numpy = _TVArray
            tvm.Tensor = _TVArray
            cumm.tensorview = tvm
            sys.modules['cumm'] = cumm
            sys.modules['cumm.tensorview'] = tvm
    return pkg
