"""The five inference modules of the plane-sweep depth path (+ their building blocks) behind the reference's class
names, constructor / forward signatures and state-dict keys (reference dvmvs/fusionnet/model.py:15-337,
dvmvs/pairnet/model.py; key contract: SURVEY.md App. C), so the shipped weight files load with strict=True.

nn.Conv2d / nn.BatchNorm2d objects are parameter holders only.  forward() runs BatchNorm-folded weights through
libdvmvs_sm90.so: channel-last activations, torch.cat fused into the conv loader as a K-split over sources,
x2 bilinear upsampling fused into the loader, FPN top-down add and MnasNet residual adds fused into the conv
epilogue, sigmoid depth heads emitting the depth map in the same launch.  Tensors handed back to the caller are
(B,C,H,W)-shaped fp32 views with channels_last strides.
"""
import torch

from . import _native as N
from . import _ops as ops
from ._base import NativeModule, auto_graph, pack_cbr, pack_head
from .config import Config
from .convlstm import MVSLayernormConvLSTMCell
from .layers import conv_layer, depth_layer_3x3

fpn_output_channels = 32
hyper_channels = 32

D, U = N.SRC_DIRECT, N.SRC_UPSAMPLE2X


# ------------------------------------------------------------------------------------------ building blocks
class StandardLayer(NativeModule):
    def __init__(self, channels, kernel_size, apply_bn_relu):
        super().__init__()
        self.conv1 = conv_layer(channels, channels, kernel_size, 1, True)
        self.conv2 = conv_layer(channels, channels, kernel_size, 1, apply_bn_relu)

    def _pack(self):
        return ops.ConvLayer(pack_cbr(self.conv1)), ops.ConvLayer(pack_cbr(self.conv2))

    def run(self, x):
        c1, c2 = self.packed()
        return c2.run([(c1.run([(x, D)]), D)])

    def forward(self, x):
        return ops.act_to_api(self.run(ops.to_act(x)))


class DownconvolutionLayer(NativeModule):
    def __init__(self, input_channels, output_channels, kernel_size):
        super().__init__()
        self.down_conv = conv_layer(input_channels, output_channels, kernel_size, 2, True)

    def _pack(self):
        return ops.ConvLayer(pack_cbr(self.down_conv, stride=2))

    def run(self, x):
        return self.packed().run([(x, D)])

    def forward(self, x):
        return ops.act_to_api(self.run(ops.to_act(x)))


class UpconvolutionLayer(NativeModule):
    def __init__(self, input_channels, output_channels, kernel_size):
        super().__init__()
        self.conv = conv_layer(input_channels, output_channels, kernel_size, 1, True)

    def _pack(self):
        return ops.ConvLayer(pack_cbr(self.conv))

    def run(self, x):
        return self.packed().run([(x, U)])                # F.interpolate(x2, bilinear, align_corners) fused / staged by the loader

    def forward(self, x):
        return ops.act_to_api(self.run(ops.to_act(x)))


class EncoderBlock(NativeModule):
    def __init__(self, input_channels, output_channels, kernel_size):
        super().__init__()
        self.down_convolution = DownconvolutionLayer(input_channels, output_channels, kernel_size)
        self.standard_convolution = StandardLayer(output_channels, kernel_size, True)

    def _pack(self):
        return ()

    def run(self, x):
        return self.standard_convolution.run(self.down_convolution.run(x))

    def forward(self, x):
        return ops.act_to_api(self.run(ops.to_act(x)))


class DecoderBlock(NativeModule):
    def __init__(self, input_channels, output_channels, kernel_size, apply_bn_relu, plus_one):
        super().__init__()
        self.plus_one = plus_one
        self.up_convolution = UpconvolutionLayer(input_channels, output_channels, kernel_size)
        self.convolution1 = conv_layer(input_channels + 1 if plus_one else input_channels, output_channels, kernel_size, 1, True)
        self.convolution2 = conv_layer(output_channels, output_channels, kernel_size, 1, apply_bn_relu)

    def _pack(self):
        cout = self.convolution2[0].in_channels
        split = [cout, self.convolution1[0].in_channels - cout - (1 if self.plus_one else 0)] + ([1] if self.plus_one else [])
        return ops.ConvLayer(pack_cbr(self.convolution1), split), ops.ConvLayer(pack_cbr(self.convolution2))

    def run(self, x, skip, depth, depth_producer=None):
        """depth_producer: callable returning the depth Act (the previous scale's sigmoid head) -- run on a side stream
        together with the staging of its x2-upsampled operand, next to the up-convolution (they are independent)."""
        c1, c2 = self.packed()
        fork = None
        if depth_producer is not None:
            fork = ops.Fork()
            with fork:
                depth = depth_producer()
                c1.prestage_upsampled(depth)
        x = self.up_convolution.run(x)
        if fork is not None:
            fork.join()
        srcs = [(x, D), (skip, D)] if depth is None else [(x, D), (skip, D), (depth, U)]   # cat fused (model.py:112-115)
        # conv1's output is read only by conv2: on the halo path that is just the blocked planes.  The block's output is read
        # as fp32 (the depth head, the next block's x2-upsampling loader, the API), so conv2 writes fp32 only.
        h, w = x.f32.shape[1], x.f32.shape[2]
        blk_only = c1.path(h, w) == "halo" and c2.path(h, w) == "halo"
        y = c1.run(srcs, want_f32=not blk_only, want_planes=not blk_only)
        return c2.run([(y, D)], want_planes=False, want_blk=False)

    def forward(self, x, skip, depth):
        return ops.act_to_api(self.run(ops.to_act(x), ops.to_act(skip), None if depth is None else ops.to_act(depth)))


# ------------------------------------------------------------------------------------------ MnasNet-1.0 trunk
class _InvertedResidual(torch.nn.Module):
    """Holder with torchvision's `_InvertedResidual` key layout: layers.{0,3,6} convs, layers.{1,4,7} BatchNorms."""

    def __init__(self, in_ch, out_ch, kernel_size, stride, expansion):
        super().__init__()
        mid = in_ch * expansion
        self.apply_residual = in_ch == out_ch and stride == 1
        self.stride = stride
        self.layers = torch.nn.Sequential(
            torch.nn.Conv2d(in_ch, mid, 1, bias=False), torch.nn.BatchNorm2d(mid), torch.nn.ReLU(inplace=True),
            torch.nn.Conv2d(mid, mid, kernel_size, padding=kernel_size // 2, stride=stride, groups=mid, bias=False),
            torch.nn.BatchNorm2d(mid), torch.nn.ReLU(inplace=True),
            torch.nn.Conv2d(mid, out_ch, 1, bias=False), torch.nn.BatchNorm2d(out_ch))


def _stack(in_ch, out_ch, kernel_size, stride, expansion, repeats):
    blocks = [_InvertedResidual(in_ch, out_ch, kernel_size, stride, expansion)]
    blocks += [_InvertedResidual(out_ch, out_ch, kernel_size, 1, expansion) for _ in range(repeats - 1)]
    return torch.nn.Sequential(*blocks)


class FeatureExtractor(NativeModule):
    """MnasNet-1.0 layers[0:14] (what torchvision.models.mnasnet1_0().layers holds; SURVEY.md App. A.5), built locally so
    construction never touches the network.  forward(image) -> (layer1..layer5) at 1/2 .. 1/32 resolution."""

    def __init__(self):
        super().__init__()
        self.layer1 = torch.nn.Sequential(
            torch.nn.Conv2d(3, 32, 3, padding=1, stride=2, bias=False), torch.nn.BatchNorm2d(32), torch.nn.ReLU(inplace=True),
            torch.nn.Conv2d(32, 32, 3, padding=1, stride=1, groups=32, bias=False), torch.nn.BatchNorm2d(32), torch.nn.ReLU(inplace=True),
            torch.nn.Conv2d(32, 16, 1, padding=0, stride=1, bias=False), torch.nn.BatchNorm2d(16))
        self.layer2 = torch.nn.Sequential(_stack(16, 24, 3, 2, 3, 3))
        self.layer3 = torch.nn.Sequential(_stack(24, 40, 5, 2, 3, 3))
        self.layer4 = torch.nn.Sequential(_stack(40, 80, 5, 2, 6, 3), _stack(80, 96, 3, 1, 6, 2))
        self.layer5 = torch.nn.Sequential(_stack(96, 192, 5, 2, 6, 4), _stack(192, 320, 3, 1, 6, 1))

    def _pack(self):
        l1 = self.layer1
        stem = (ops.ConvLayer(ops.PackedConv(l1[0].weight, None, l1[1], stride=2, act=N.ACT_RELU)),
                ops.PackedDepthwise(l1[3].weight, l1[4], stride=1),
                ops.ConvLayer(ops.PackedConv(l1[6].weight, None, l1[7], stride=1, act=N.ACT_NONE)))
        levels = []
        for layer in (self.layer2, self.layer3, self.layer4, self.layer5):
            blocks = []
            for stack in layer:
                for blk in stack:
                    L = blk.layers
                    blocks.append((ops.ConvLayer(ops.PackedConv(L[0].weight, None, L[1], act=N.ACT_RELU)),
                                   ops.PackedDepthwise(L[3].weight, L[4], stride=blk.stride),
                                   ops.ConvLayer(ops.PackedConv(L[6].weight, None, L[7], act=N.ACT_NONE)), blk.apply_residual))
            levels.append(blocks)
        return stem, levels

    def run(self, x, image_nchw=None, part="all"):
        """part: "all" -> [layer1..layer5]; "head" -> [layer1, layer2, layer3]; "tail" (x = layer3 Act) -> [layer4, layer5]."""
        stem, levels = self.packed()
        def depthwise(t, dw, consumer):
            # the depthwise output feeds exactly one pointwise conv: hand it the operand format that conv reads
            if consumer.uses_tc():
                return ops.Act(None, ops.dwconv2d(t.f32, dw, want_f32=False, want_planes=True)[1])
            return ops.Act(ops.dwconv2d(t.f32, dw))

        outs = []
        if part != "tail":
            if image_nchw is not None:        # dedicated stem kernel reads the NCHW image directly (no layout pass)
                x = ops.Act(ops.stem_conv(image_nchw, stem[0].pc))
            else:
                x = stem[0].run([(x, D)])
            x = depthwise(x, stem[1], stem[2])
            x = stem[2].run([(x, D)])
            outs = [x]
        for blocks in {"all": levels, "head": levels[:2], "tail": levels[2:]}[part]:
            for expand, dw, project, residual in blocks:
                if expand.uses_tc():
                    # expansion + depthwise in one launch: the expanded tensor never leaves shared memory
                    y = ops.Act(None, ops.expand_dwconv(x, expand, dw))
                else:
                    y = depthwise(expand.run([(x, D)], want_planes=False), dw, project)
                x = project.run([(y, D)], residual=x if residual else None,
                                residual_mode=N.RES_SAME if residual else N.RES_NONE)
            outs.append(x)
        return outs

    @auto_graph
    @ops.family_terms("fe")
    def forward(self, image):
        B, C, H, W = image.shape
        if C != 3 or H % 32 != 0 or W % 32 != 0:
            raise RuntimeError("FeatureExtractor: expected (B,3,H,W) with H, W multiples of 32, got %s" % (tuple(image.shape),))
        ops.require_cuda_f32(image, "image")
        if image.is_contiguous():
            return tuple(ops.act_to_api(t) for t in self.run(None, image_nchw=image))
        return tuple(ops.act_to_api(t) for t in self.run(ops.to_act(image, "image")))

    @ops.family_terms("fe")
    def forward_head(self, image):
        """layer1..layer3 only (pipeline engines split the trunk here); forward_tail(head) completes it."""
        ops.require_cuda_f32(image, "image")
        return tuple(ops.act_to_api(t) for t in self.run(None, image_nchw=image.contiguous(), part="head"))

    @ops.family_terms("fe")
    def forward_tail(self, head):
        l1, l2, l3 = head
        tail = self.run(ops.to_act(l3, "layer3"), part="tail")
        return (l1, l2, l3) + tuple(ops.act_to_api(t) for t in tail)


class _FPNHolder(torch.nn.Module):
    """torchvision FeaturePyramidNetwork parameters under the flat keys the shipped files use
    (fpn.inner_blocks.{i}.{weight,bias}, fpn.layer_blocks.{i}.{weight,bias})."""

    def __init__(self, in_channels_list, out_channels):
        super().__init__()
        self.inner_blocks = torch.nn.ModuleList([torch.nn.Conv2d(c, out_channels, 1) for c in in_channels_list])
        self.layer_blocks = torch.nn.ModuleList([torch.nn.Conv2d(out_channels, out_channels, 3, padding=1) for _ in in_channels_list])


class FeatureShrinker(NativeModule):
    """FPN([16,24,40,96,320] -> 32): 1x1 lateral convs, top-down nearest-upsample add fused into the lateral conv's
    epilogue, 3x3 output convs.  The level-5 output conv (computed and discarded by the reference, model.py:159-162) is
    skipped."""

    def __init__(self):
        super().__init__()
        self.fpn = _FPNHolder([16, 24, 40, 96, 320], fpn_output_channels)

    def _pack(self):
        inner = [ops.ConvLayer(ops.PackedConv(m.weight, m.bias)) for m in self.fpn.inner_blocks]
        layer = [ops.ConvLayer(ops.PackedConv(m.weight, m.bias)) for m in self.fpn.layer_blocks]
        return inner, layer

    def run(self, feats):
        inner, layer = self.packed()
        last = inner[4].run([(feats[4], D)])
        outs = [None] * 4
        keep, forks = [last], []          # tensors read on the side stream stay referenced until the joins
        for i in (3, 2, 1, 0):
            last = inner[i].run([(feats[i], D)], residual=last, residual_mode=N.RES_NEAREST_UP)
            keep.append(last)
            if i > 0:
                # the 3x3 output conv of level i is off the top-down chain (inner[i-1] only needs `last`): side stream
                f = ops.Fork()
                with f:
                    outs[i] = layer[i].run([(last, D)])
                forks.append(f)
            else:
                outs[i] = layer[i].run([(last, D)])
        for f in forks:
            f.join()
        del keep
        return outs

    @auto_graph
    @ops.family_terms("fpn")
    def forward(self, layer1, layer2, layer3, layer4, layer5):
        feats = [ops.to_act(t, "layer%d" % (i + 1)) for i, t in enumerate((layer1, layer2, layer3, layer4, layer5))]
        return tuple(ops.act_to_api(t) for t in self.run(feats))


# ------------------------------------------------------------------------------------------ cost-volume encoder / decoder
class CostVolumeEncoder(NativeModule):
    def __init__(self):
        super().__init__()
        h = hyper_channels
        self.aggregator0 = conv_layer(Config.train_n_depth_levels + fpn_output_channels, h, 5, 1, True)
        self.encoder_block0 = EncoderBlock(h, h * 2, 5)
        self.aggregator1 = conv_layer(h * 2 + fpn_output_channels, h * 2, 3, 1, True)
        self.encoder_block1 = EncoderBlock(h * 2, h * 4, 3)
        self.aggregator2 = conv_layer(h * 4 + fpn_output_channels, h * 4, 3, 1, True)
        self.encoder_block2 = EncoderBlock(h * 4, h * 8, 3)
        self.aggregator3 = conv_layer(h * 8 + fpn_output_channels, h * 8, 3, 1, True)
        self.encoder_block3 = EncoderBlock(h * 8, h * 16, 3)

    def _pack(self):
        return [ops.ConvLayer(pack_cbr(a), [fpn_output_channels, a[0].in_channels - fpn_output_channels])
                for a in (self.aggregator0, self.aggregator1, self.aggregator2, self.aggregator3)]

    def run(self, f2, f4, f8, f16, cost_volume):
        agg = self.packed()
        inp0 = agg[0].run([(f2, D), (cost_volume, D)])                      # cat order model.py:208
        out0 = self.encoder_block0.run(inp0)
        inp1 = agg[1].run([(f4, D), (out0, D)])
        out1 = self.encoder_block1.run(inp1)
        inp2 = agg[2].run([(f8, D), (out1, D)])
        out2 = self.encoder_block2.run(inp2)
        inp3 = agg[3].run([(f16, D), (out2, D)])
        out3 = self.encoder_block3.run(inp3)
        return inp0, inp1, inp2, inp3, out3

    @auto_graph
    @ops.family_terms("cve")
    def forward(self, features_half, features_quarter, features_one_eight, features_one_sixteen, cost_volume):
        args = [ops.to_act(t, n) for t, n in ((features_half, "features_half"), (features_quarter, "features_quarter"),
                                              (features_one_eight, "features_one_eight"),
                                              (features_one_sixteen, "features_one_sixteen"), (cost_volume, "cost_volume"))]
        return tuple(ops.act_to_api(t) for t in self.run(*args))


class CostVolumeDecoder(NativeModule):
    def __init__(self):
        super().__init__()
        h = hyper_channels
        self.inverse_depth_base = 1 / Config.train_max_depth
        self.inverse_depth_multiplier = 1 / Config.train_min_depth - 1 / Config.train_max_depth
        self.decoder_block1 = DecoderBlock(h * 16, h * 8, 3, True, False)
        self.decoder_block2 = DecoderBlock(h * 8, h * 4, 3, True, True)
        self.decoder_block3 = DecoderBlock(h * 4, h * 2, 3, True, True)
        self.decoder_block4 = DecoderBlock(h * 2, h, 5, True, True)
        self.refine = torch.nn.Sequential(conv_layer(h + 4, h, 5, 1, True), conv_layer(h, h, 5, 1, True))
        self.depth_layer_one_sixteen = depth_layer_3x3(h * 8)
        self.depth_layer_one_eight = depth_layer_3x3(h * 4)
        self.depth_layer_quarter = depth_layer_3x3(h * 2)
        self.depth_layer_half = depth_layer_3x3(h)
        self.depth_layer_full = depth_layer_3x3(h)

    def _pack(self):
        heads = [ops.ConvLayer(pack_head(m)) for m in (self.depth_layer_one_sixteen, self.depth_layer_one_eight,
                                                       self.depth_layer_quarter, self.depth_layer_half, self.depth_layer_full)]
        return heads, ops.ConvLayer(pack_cbr(self.refine[0]), [hyper_channels, 1, 3], pack_sources=True), ops.ConvLayer(pack_cbr(self.refine[1]))

    def run(self, image, skip0, skip1, skip2, skip3, bottom):
        heads, r0, r1 = self.packed()
        aux = (float(self.inverse_depth_multiplier), float(self.inverse_depth_base))    # depth = 1/(mult*sigmoid + base)
        depths = {}

        def head(i, d):
            # scale-i depth head; returns the sigmoid map the next block concatenates, keeps the depth output
            def produce():
                sig, depths[i] = heads[i].run([(d, D)], aux=aux)
                return sig
            return produce

        # each head (+ the staging of its upsampled output) is independent of the next block's up-convolution: fork / join
        d1 = self.decoder_block1.run(bottom, skip3, None)
        d2 = self.decoder_block2.run(d1, skip2, None, depth_producer=head(0, d1))
        d3 = self.decoder_block3.run(d2, skip1, None, depth_producer=head(1, d2))
        d4 = self.decoder_block4.run(d3, skip0, None, depth_producer=head(2, d3))
        Ho, Wo = 2 * d4.f32.shape[1], 2 * d4.f32.shape[2]
        # refine.0's output is read only by refine.1 (on the halo path: its blocked planes); refine.1's only by the fp32 depth head
        r0_out = {"want_f32": False, "want_planes": False} if r0.path(Ho, Wo) == "halo" and r1.path(Ho, Wo) == "halo" else {}
        if r0.pack_sources and r0.path(Ho, Wo) == "halo":
            # refine.0 reads ONE concatenated operand [up(d4), up(sigmoid), image]: the head runs on the side stream while
            # the two sources that exist already are staged; the sigmoid map is staged after the join
            fork = ops.Fork()
            with fork:
                s2 = head(3, d4)()
            meta = [(d4.f32, True), ((d4.f32.shape[0], d4.f32.shape[1], d4.f32.shape[2], 1), True), (image.f32, False)]
            buf = ops.split_blocked(meta, only=(0, 2))
            fork.join()
            ops.split_blocked([(d4.f32, True), (s2.f32, True), (image.f32, False)], only=(1,), into=buf)
            x = r0.run([(d4, U), (s2, U), (image, D)], prestaged=buf, **r0_out)           # cat order model.py:295
        else:
            s2 = head(3, d4)()
            x = r0.run([(d4, U), (s2, U), (image, D)], **r0_out)                          # cat order model.py:295
        depth16, depth8, depth4, depth2 = depths[0], depths[1], depths[2], depths[3]
        x = r1.run([(x, D)], want_planes=False, want_blk=False)
        _, depth1 = heads[4].run([(x, D)], aux=aux)
        return [t.squeeze(3) for t in (depth1, depth2, depth4, depth8, depth16)]

    @auto_graph
    @ops.family_terms("cvd")
    def forward(self, image, skip0, skip1, skip2, skip3, bottom):
        args = [ops.to_act(t, n) for t, n in ((image, "image"), (skip0, "skip0"), (skip1, "skip1"), (skip2, "skip2"),
                                              (skip3, "skip3"), (bottom, "bottom"))]
        return tuple(self.run(*args))


class LSTMFusion(NativeModule):
    def __init__(self):
        super().__init__()
        self.lstm_cell = MVSLayernormConvLSTMCell(input_dim=hyper_channels * 16, hidden_dim=hyper_channels * 16,
                                                  kernel_size=(3, 3), activation_function=torch.celu)

    def _pack(self):
        return ()

    @auto_graph
    @ops.family_terms("lstm")
    def forward(self, current_encoding, current_state, previous_pose, current_pose, estimated_current_depth, camera_matrix,
                input_gates=None):
        """input_gates (optional, beyond the reference signature): lstm_cell.input_gates(current_encoding) computed earlier."""
        batch, channel, height, width = current_encoding.size()
        if current_state is None:                                                        # model.py:324-326
            current_state = self.lstm_cell.init_hidden(batch_size=batch, image_size=(height, width))
        return self.lstm_cell(input_tensor=current_encoding, cur_state=list(current_state), previous_pose=previous_pose,
                              current_pose=current_pose, estimated_current_depth=estimated_current_depth,
                              camera_matrix=camera_matrix, input_gates=input_gates)
