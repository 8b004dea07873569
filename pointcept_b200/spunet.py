"""SpUNet-v1m1 on the CUDA sparse-conv operators: host-side mirror of
pointcept/models/sparse_unet/spconv_unet_v1m1_base.py:23-280 (same module tree / parameter names)."""
from collections import OrderedDict
from functools import partial

import torch
import torch.nn as nn

from .spconv import pytorch as spconv


class BasicBlock(spconv.SparseModule):
    expansion = 1

    def __init__(self, in_channels, embed_channels, stride=1, norm_fn=None, indice_key=None, bias=False):
        super().__init__()
        assert norm_fn is not None
        if in_channels == embed_channels:
            self.proj = spconv.SparseSequential(nn.Identity())
        else:
            self.proj = spconv.SparseSequential(spconv.SubMConv3d(in_channels, embed_channels, kernel_size=1, bias=False),
                                                norm_fn(embed_channels))
        self.conv1 = spconv.SubMConv3d(in_channels, embed_channels, kernel_size=3, stride=stride, padding=1, bias=bias,
                                       indice_key=indice_key)
        self.bn1 = norm_fn(embed_channels)
        self.relu = nn.ReLU()
        self.conv2 = spconv.SubMConv3d(embed_channels, embed_channels, kernel_size=3, stride=stride, padding=1, bias=bias,
                                       indice_key=indice_key)
        self.bn2 = norm_fn(embed_channels)
        self.stride = stride

    def forward(self, x):
        out = self.conv1(x)
        out = out.replace_feature(self.relu(self.bn1(out.features)))
        out = self.conv2(out)
        out = out.replace_feature(self.bn2(out.features))
        out = out.replace_feature(self.relu(out.features + self.proj(x).features))
        return out


class SpUNetBase(nn.Module):
    """ "SpUNet-v1m1" with the reference's constructor arguments."""

    def __init__(self, in_channels, num_classes, base_channels=32, channels=(32, 64, 128, 256, 256, 128, 96, 96),
                 layers=(2, 3, 4, 6, 2, 2, 2, 2), enc_mode=False):
        super().__init__()
        assert len(layers) % 2 == 0 and len(layers) == len(channels)
        self.in_channels, self.num_classes, self.base_channels = in_channels, num_classes, base_channels
        self.channels, self.layers, self.num_stages, self.enc_mode = channels, layers, len(layers) // 2, enc_mode
        norm_fn = partial(nn.BatchNorm1d, eps=1e-3, momentum=0.01)
        self.conv_input = spconv.SparseSequential(
            spconv.SubMConv3d(in_channels, base_channels, kernel_size=5, padding=1, bias=False, indice_key="stem"),
            norm_fn(base_channels), nn.ReLU())
        enc_channels, dec_channels = base_channels, channels[-1]
        self.down, self.up, self.enc = nn.ModuleList(), nn.ModuleList(), nn.ModuleList()
        self.dec = nn.ModuleList() if not enc_mode else None
        for s in range(self.num_stages):
            self.down.append(spconv.SparseSequential(
                spconv.SparseConv3d(enc_channels, channels[s], kernel_size=2, stride=2, bias=False, indice_key=f"spconv{s + 1}"),
                norm_fn(channels[s]), nn.ReLU()))
            self.enc.append(spconv.SparseSequential(OrderedDict(
                (f"block{i}", BasicBlock(channels[s], channels[s], norm_fn=norm_fn, indice_key=f"subm{s + 1}"))
                for i in range(layers[s]))))
            if not enc_mode:
                self.up.append(spconv.SparseSequential(
                    spconv.SparseInverseConv3d(channels[len(channels) - s - 2], dec_channels, kernel_size=2, bias=False,
                                               indice_key=f"spconv{s + 1}"),
                    norm_fn(dec_channels), nn.ReLU()))
                self.dec.append(spconv.SparseSequential(OrderedDict(
                    (f"block{i}", BasicBlock(dec_channels + enc_channels if i == 0 else dec_channels, dec_channels,
                                             norm_fn=norm_fn, indice_key=f"subm{s}"))
                    for i in range(layers[len(channels) - s - 1]))))
            enc_channels = channels[s]
            dec_channels = channels[len(channels) - s - 2]
        final_in = channels[-1] if not enc_mode else channels[self.num_stages - 1]
        self.final = (spconv.SubMConv3d(final_in, num_classes, kernel_size=1, padding=1, bias=True)
                      if num_classes > 0 else spconv.Identity())
        self.apply(self._init_weights)

    @staticmethod
    def _init_weights(m):
        if isinstance(m, (nn.Linear, spconv.SubMConv3d)):
            nn.init.trunc_normal_(m.weight, std=0.02)
            if m.bias is not None:
                nn.init.constant_(m.bias, 0)
        elif isinstance(m, nn.BatchNorm1d):
            nn.init.constant_(m.bias, 0)
            nn.init.constant_(m.weight, 1.0)

    def forward(self, input_dict):
        if torch.is_autocast_enabled() and input_dict["feat"].is_cuda:
            from . import ops
            if ops.binding() is not None:      # one launch refreshes the half-precision shadows of every conv weight
                sh = self.__dict__.get("_half_shadows")
                if sh is None:
                    sh = ops.HalfShadows(self)
                    self.__dict__["_half_shadows"] = sh
                sh.sync(torch.get_autocast_dtype("cuda"))
        grid_coord, feat, offset = input_dict["grid_coord"], input_dict["feat"], input_dict["offset"]
        if "offset_host" in input_dict:
            oh = input_dict["offset_host"]
            counts = torch.tensor([b - a for a, b in zip([0] + list(oh[:-1]), oh)], device=offset.device)
            batch = torch.repeat_interleave(torch.arange(len(oh), device=offset.device), counts, output_size=int(oh[-1]))
        else:
            counts = torch.diff(offset, prepend=offset.new_zeros(1))
            batch = torch.arange(len(offset), device=offset.device).repeat_interleave(counts)
        gmax = input_dict.get("grid_max_host")
        if gmax is None:
            gmax = grid_coord.max(0).values.tolist()
        sparse_shape = [int(g) + 96 for g in gmax]
        x = spconv.SparseConvTensor(features=feat, indices=torch.cat([batch.unsqueeze(-1).int(), grid_coord.int()], dim=1).contiguous(),
                                    spatial_shape=sparse_shape, batch_size=len(offset))
        x = self.conv_input(x)
        skips = [x]
        for s in range(self.num_stages):
            x = self.enc[s](self.down[s](x))
            skips.append(x)
        x = skips.pop(-1)
        if not self.enc_mode:
            for s in reversed(range(self.num_stages)):
                x = self.up[s](x)
                skip = skips.pop(-1)
                x = x.replace_feature(torch.cat((x.features, skip.features), dim=1))
                x = self.dec[s](x)
        x = self.final(x)
        if self.enc_mode:
            idx = x.indices[:, 0].long()
            s = torch.zeros((x.batch_size, x.features.shape[1]), dtype=x.features.dtype, device=idx.device).index_add_(0, idx, x.features)
            x = x.replace_feature(s / torch.bincount(idx, minlength=x.batch_size).clamp(min=1).unsqueeze(1))
        return x.features
