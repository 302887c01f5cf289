"""HRNet-W48 backbone, host mirror of regressor/human_shape/models/backbone/hrnet.py.

Same class name, constructor argument (the `hrnet` config node), parameter tree and therefore the
same 1 967 state-dict keys as the reference module (hrnet.py:202-288), so a SHAPY_A checkpoint loads
unmodified.  nn.Conv2d / nn.BatchNorm2d objects are used purely as PARAMETER CONTAINERS: `forward`
never calls them.  Instead the module tree is compiled (lazily, and again whenever the parameters
change) into a flat program of fused conv+BN(+residual)(+ReLU) ops that the sm_90a library executes
(shapy_b200/csrc/hrnet.cu, conv_wgmma.cu).  There is no PyTorch fallback: CPU tensors raise.
"""
import os.path as osp

import torch
import torch.nn as nn

from .... import ops as _ops
from ...._lib import OP_CONV, OP_FUSE, OP_POOL, OP_STEM

BN_MOMENTUM = 0.1
N_LANES = 4          # SHAPY_MAX_LANES of include/shapy_b200.h

DEFAULT_STAGES = {  # regressor/human_shape/config/network_defaults.py:92-132
    'stage1': dict(num_modules=1, num_branches=1, num_blocks=(4,), num_channels=(64,), block='BOTTLENECK',
                   fuse_method='SUM'),
    'stage2': dict(num_modules=1, num_branches=2, num_blocks=(4, 4), num_channels=(48, 96), block='BASIC',
                   fuse_method='SUM'),
    'stage3': dict(num_modules=4, num_branches=3, num_blocks=(4, 4, 4), num_channels=(48, 96, 192), block='BASIC',
                   fuse_method='SUM'),
    'stage4': dict(num_modules=3, num_branches=4, num_blocks=(4, 4, 4, 4), num_channels=(48, 96, 192, 384),
                   block='BASIC', fuse_method='SUM'),
}


def _cfg_get(cfg, key, default=None):
    if cfg is None:
        return default
    if hasattr(cfg, 'get'):
        v = cfg.get(key, default)
    else:
        v = getattr(cfg, key, default)
    return default if v is None else v


def build(cfg, pretrained=True, **kwargs):
    hr_net_cfg = _cfg_get(cfg, 'hrnet', {})
    model = HighResolutionNet(hr_net_cfg, **kwargs)
    pretrained_path = _cfg_get(hr_net_cfg, 'pretrained_path', '')
    if pretrained and pretrained_path and osp.isfile(osp.expandvars(pretrained_path)):
        model.load_weights(pretrained_path)
    return model


def conv3x3(i, o, stride=1):
    return nn.Conv2d(i, o, kernel_size=3, stride=stride, padding=1, bias=False)


class BasicBlock(nn.Module):
    """Parameter layout of torchvision.models.resnet.BasicBlock (the reference imports it, hrnet.py:13)."""
    expansion = 1

    def __init__(self, inplanes, planes, stride=1, downsample=None):
        super().__init__()
        self.conv1 = conv3x3(inplanes, planes, stride)
        self.bn1 = nn.BatchNorm2d(planes)
        self.relu = nn.ReLU(inplace=True)
        self.conv2 = conv3x3(planes, planes)
        self.bn2 = nn.BatchNorm2d(planes)
        self.downsample = downsample
        self.stride = stride


class Bottleneck(nn.Module):
    """Parameter layout of torchvision.models.resnet.Bottleneck (stride on the 3x3)."""
    expansion = 4

    def __init__(self, inplanes, planes, stride=1, downsample=None):
        super().__init__()
        self.conv1 = nn.Conv2d(inplanes, planes, kernel_size=1, bias=False)
        self.bn1 = nn.BatchNorm2d(planes)
        self.conv2 = conv3x3(planes, planes, stride)
        self.bn2 = nn.BatchNorm2d(planes)
        self.conv3 = nn.Conv2d(planes, planes * 4, kernel_size=1, bias=False)
        self.bn3 = nn.BatchNorm2d(planes * 4)
        self.relu = nn.ReLU(inplace=True)
        self.downsample = downsample
        self.stride = stride


blocks_dict = {'BASIC': BasicBlock, 'BOTTLENECK': Bottleneck}


class HighResolutionModule(nn.Module):
    def __init__(self, num_branches, block, num_blocks, num_inchannels, num_channels, fuse_method,
                 multi_scale_output=True):
        super().__init__()
        self.num_inchannels = num_inchannels
        self.fuse_method = fuse_method
        self.num_branches = num_branches
        self.multi_scale_output = multi_scale_output
        self.branches = nn.ModuleList([
            self._make_one_branch(i, block, num_blocks, num_channels) for i in range(num_branches)])
        self.fuse_layers = self._make_fuse_layers()
        self.relu = nn.ReLU(True)

    def _make_one_branch(self, i, block, num_blocks, num_channels, stride=1):
        downsample = None
        if stride != 1 or self.num_inchannels[i] != num_channels[i] * block.expansion:
            downsample = nn.Sequential(
                nn.Conv2d(self.num_inchannels[i], num_channels[i] * block.expansion, kernel_size=1, stride=stride,
                          bias=False),
                nn.BatchNorm2d(num_channels[i] * block.expansion, momentum=BN_MOMENTUM))
        layers = [block(self.num_inchannels[i], num_channels[i], stride, downsample)]
        self.num_inchannels[i] = num_channels[i] * block.expansion
        for _ in range(1, num_blocks[i]):
            layers.append(block(self.num_inchannels[i], num_channels[i]))
        return nn.Sequential(*layers)

    def _make_fuse_layers(self):
        if self.num_branches == 1:
            return None
        nb, nin = self.num_branches, self.num_inchannels
        fuse_layers = []
        for i in range(nb if self.multi_scale_output else 1):
            fuse_layer = []
            for j in range(nb):
                if j > i:
                    fuse_layer.append(nn.Sequential(
                        nn.Conv2d(nin[j], nin[i], 1, 1, 0, bias=False), nn.BatchNorm2d(nin[i]),
                        nn.Upsample(scale_factor=2 ** (j - i), mode='nearest')))
                elif j == i:
                    fuse_layer.append(None)
                else:
                    convs = []
                    for k in range(i - j):
                        if k == i - j - 1:
                            convs.append(nn.Sequential(nn.Conv2d(nin[j], nin[i], 3, 2, 1, bias=False),
                                                       nn.BatchNorm2d(nin[i])))
                        else:
                            convs.append(nn.Sequential(nn.Conv2d(nin[j], nin[j], 3, 2, 1, bias=False),
                                                       nn.BatchNorm2d(nin[j]), nn.ReLU(True)))
                    fuse_layer.append(nn.Sequential(*convs))
            fuse_layers.append(nn.ModuleList(fuse_layer))
        return nn.ModuleList(fuse_layers)

    def get_num_inchannels(self):
        return self.num_inchannels


class _Graph:
    """Flat op program over virtual tensors; physical slots are assigned by liveness afterwards."""

    def __init__(self):
        self.convs, self.ops, self.tensors = [], [], []
        self.keep = set()
        self.lane = 0       # execution lane of the ops emitted next (scheduling hint, see shapy_op_t.lane)

    def on(self, lane):
        self.lane = int(lane) % N_LANES
        return self

    def tensor(self, channels, div):
        self.tensors.append(dict(channels=channels, div=div, lane=self.lane))
        return len(self.tensors) - 1

    def _conv_entry(self, conv, bn):
        e = dict(cin=conv.in_channels, cout=conv.out_channels, ksize=conv.kernel_size[0], stride=conv.stride[0],
                 weight=conv.weight, bias=conv.bias, bn=None)
        if bn is not None:
            e['bn'] = dict(weight=bn.weight, bias=bn.bias, mean=bn.running_mean, var=bn.running_var, eps=bn.eps)
        self.convs.append(e)
        return len(self.convs) - 1

    def conv(self, conv, bn, x, relu, res=None, out=None, out_coff=0):
        div = self.tensors[x]['div'] * conv.stride[0] if x >= 0 else conv.stride[0]
        if out is None:
            out = self.tensor(conv.out_channels, div)
        self.ops.append(dict(kind=OP_STEM if x < 0 else OP_CONV, conv=self._conv_entry(conv, bn), in_slot=x,
                             out_slot=out, out_coff=out_coff, res_slot=-1 if res is None else res, relu=int(relu),
                             lane=self.lane))
        return out

    def fuse(self, ins, relu=True):
        t0 = self.tensors[ins[0][0]]
        out = self.tensor(t0['channels'], t0['div'] >> ins[0][1])
        self.ops.append(dict(kind=OP_FUSE, out_slot=out, relu=int(relu), fuse_in=[t for t, _ in ins],
                             fuse_shift=[s for _, s in ins], lane=self.lane))
        return out

    def pool(self, x):
        self.ops.append(dict(kind=OP_POOL, in_slot=x, lane=self.lane))

    def finalize(self):
        """Liveness-based slot reuse.  Returns (ops with physical slots, slots, virtual->physical map)."""
        def reads(o):
            r = []
            if o['kind'] in (OP_CONV, OP_POOL) and o.get('in_slot', -1) >= 0:
                r.append(o['in_slot'])
            if o.get('res_slot', -1) >= 0:
                r.append(o['res_slot'])
            r += o.get('fuse_in', [])
            return r
        last = {}
        for i, o in enumerate(self.ops):
            for t in reads(o):
                last[t] = i
            if 'out_slot' in o:
                last.setdefault(o['out_slot'], i)
                last[o['out_slot']] = max(last[o['out_slot']], i)
        phys, slots, free = {}, [], {}
        out_ops = []
        for i, o in enumerate(self.ops):
            o = dict(o)
            if 'out_slot' in o and o['out_slot'] not in phys:
                t = self.tensors[o['out_slot']]
                # slots are only recycled within a lane: a recycled slot orders its new writer after the old readers
                # (WAR), which across lanes would serialise branches that are independent
                key = (t['channels'], t['div'], t['lane'])
                # never alias an op's output with one of its own inputs
                busy = {phys[r] for r in reads(o) if r in phys}
                cand = [s for s in free.get(key, []) if s not in busy]
                if cand:
                    s = cand[0]
                    free[key].remove(s)
                else:
                    slots.append(dict(channels=t['channels'], div=t['div']))
                    s = len(slots) - 1
                phys[o['out_slot']] = s
            for k in ('in_slot', 'res_slot', 'out_slot'):
                if o.get(k, -1) >= 0:
                    o[k] = phys[o[k]]
            if 'fuse_in' in o:
                o['fuse_in'] = [phys[t] for t in o['fuse_in']]
            out_ops.append(o)
            for t in set(reads(self.ops[i]) + ([self.ops[i]['out_slot']] if 'out_slot' in self.ops[i] else [])):
                if last.get(t) == i and t not in self.keep and t in phys:
                    tt = self.tensors[t]
                    free.setdefault((tt['channels'], tt['div'], tt['lane']), []).append(phys[t])
        return out_ops, slots, phys


class _Outputs(dict):
    """output dict of HighResolutionNet.forward: 'concat' is materialised, 'layerN' on first access."""

    def __init__(self, plan, layer_slots, concat):
        super().__init__(concat=concat)
        self._plan, self._layer_slots = plan, layer_slots

    def __missing__(self, key):
        if key in self._layer_slots:
            v = self._plan.read_slot(self._layer_slots[key])
            self[key] = v
            return v
        raise KeyError(key)

    def keys(self):
        return list(self._layer_slots) + ['concat']

    def __contains__(self, key):
        return key == 'concat' or key in self._layer_slots


class HighResolutionNet(nn.Module):
    # numeric mode of the compiled plan: 1 = split-fp16 parity mode (fp32-grade), 0 = plain fp16 operands
    precision_mode = 1
    engine = 0      # 0 = wgmma implicit GEMM, 1 = SIMT fp32 (debug cross-check)

    def __init__(self, cfg=None, **kwargs):
        self.inplanes = 64
        super().__init__()
        use_old_impl = bool(_cfg_get(cfg, 'use_old_impl', False))
        if use_old_impl:
            raise ValueError('shapy_b200: use_old_impl=True is not on the SHAPY_A path')
        self.use_old_impl = use_old_impl
        self.conv1 = nn.Conv2d(3, 64, kernel_size=3, stride=2, padding=1, bias=False)
        self.bn1 = nn.BatchNorm2d(64, momentum=BN_MOMENTUM)
        self.conv2 = nn.Conv2d(64, 64, kernel_size=3, stride=2, padding=1, bias=False)
        self.bn2 = nn.BatchNorm2d(64, momentum=BN_MOMENTUM)
        self.relu = nn.ReLU(inplace=True)

        def stage_cfg(name):
            s = _cfg_get(cfg, name, None)
            d = dict(DEFAULT_STAGES[name])
            if s is not None:
                for k in d:
                    d[k] = _cfg_get(s, k, d[k])
            return d

        self.stage1_cfg = stage_cfg('stage1')
        num_channels = self.stage1_cfg['num_channels'][0]
        block = blocks_dict[self.stage1_cfg['block']]
        self.layer1 = self._make_layer(block, num_channels, self.stage1_cfg['num_blocks'][0])
        stage1_out_channel = block.expansion * num_channels

        self.stage2_cfg = stage_cfg('stage2')
        block = blocks_dict[self.stage2_cfg['block']]
        num_channels = [c * block.expansion for c in self.stage2_cfg['num_channels']]
        stage2_num_channels = num_channels
        self.transition1 = self._make_transition_layer([stage1_out_channel], num_channels)
        self.stage2, pre = self._make_stage(self.stage2_cfg, num_channels)

        self.stage3_cfg = stage_cfg('stage3')
        block = blocks_dict[self.stage3_cfg['block']]
        num_channels = [c * block.expansion for c in self.stage3_cfg['num_channels']]
        stage3_num_channels = num_channels
        self.transition2 = self._make_transition_layer(pre, num_channels)
        self.stage3, pre = self._make_stage(self.stage3_cfg, num_channels)

        self.stage4_cfg = stage_cfg('stage4')
        block = blocks_dict[self.stage4_cfg['block']]
        num_channels = [c * block.expansion for c in self.stage4_cfg['num_channels']]
        self.transition3 = self._make_transition_layer(pre, num_channels)
        self.stage4, pre = self._make_stage(self.stage4_cfg, num_channels, multi_scale_output=True)
        stage4_num_channels = num_channels
        self.output_channels_dim = pre
        self.pretrained_layers = _cfg_get(cfg, 'pretrained_layers', ('*',))
        self.init_weights()
        self.avg_pooling = nn.AdaptiveAvgPool2d(1)
        in_dims = 4 * 384
        self.subsample_4 = self._make_subsample_layer(in_channels=stage4_num_channels[0], num_layers=3)
        self.subsample_3 = self._make_subsample_layer(in_channels=stage2_num_channels[-1], num_layers=2)
        self.subsample_2 = self._make_subsample_layer(in_channels=stage3_num_channels[-1], num_layers=1)
        self.conv_layers = self._make_conv_layer(in_channels=in_dims, num_layers=5)
        self._plan = None
        self._plan_key = None

    # ------------------------------------------------------------------ construction (hrnet.py:301-424)
    def get_output_dim(self):
        base = {f'layer{i + 1}': v for i, v in enumerate(self.output_channels_dim)}
        out = dict(base)
        for k in base:
            out[f'{k}_avg_pooling'] = out[k]
        out['concat'] = 2048
        return out

    def _make_transition_layer(self, pre, cur):
        layers = []
        for i in range(len(cur)):
            if i < len(pre):
                if cur[i] != pre[i]:
                    layers.append(nn.Sequential(nn.Conv2d(pre[i], cur[i], 3, 1, 1, bias=False),
                                                nn.BatchNorm2d(cur[i]), nn.ReLU(inplace=True)))
                else:
                    layers.append(None)
            else:
                convs = []
                for j in range(i + 1 - len(pre)):
                    inc = pre[-1]
                    outc = cur[i] if j == i - len(pre) else inc
                    convs.append(nn.Sequential(nn.Conv2d(inc, outc, 3, 2, 1, bias=False), nn.BatchNorm2d(outc),
                                               nn.ReLU(inplace=True)))
                layers.append(nn.Sequential(*convs))
        return nn.ModuleList(layers)

    def _make_layer(self, block, planes, blocks, stride=1):
        downsample = None
        if stride != 1 or self.inplanes != planes * block.expansion:
            downsample = nn.Sequential(
                nn.Conv2d(self.inplanes, planes * block.expansion, kernel_size=1, stride=stride, bias=False),
                nn.BatchNorm2d(planes * block.expansion, momentum=BN_MOMENTUM))
        layers = [block(self.inplanes, planes, stride, downsample)]
        self.inplanes = planes * block.expansion
        for _ in range(1, blocks):
            layers.append(block(self.inplanes, planes))
        return nn.Sequential(*layers)

    def _make_conv_layer(self, in_channels=2048, num_layers=3, num_filters=2048, stride=1):
        layers = []
        for _ in range(num_layers):
            downsample = nn.Conv2d(in_channels, num_filters, stride=1, kernel_size=1, bias=False)
            layers.append(Bottleneck(in_channels, num_filters // 4, downsample=downsample))
            in_channels = num_filters
        return nn.Sequential(*layers)

    def _make_subsample_layer(self, in_channels=96, num_layers=3, stride=2):
        layers = []
        for _ in range(num_layers):
            layers.append(nn.Conv2d(in_channels, 2 * in_channels, kernel_size=3, stride=stride, padding=1))
            in_channels = 2 * in_channels
            layers.append(nn.BatchNorm2d(in_channels, momentum=BN_MOMENTUM))
            layers.append(nn.ReLU(inplace=True))
        return nn.Sequential(*layers)

    def _make_stage(self, layer_config, num_inchannels, multi_scale_output=True):
        block = blocks_dict[layer_config['block']]
        modules = []
        for i in range(layer_config['num_modules']):
            reset = not (not multi_scale_output and i == layer_config['num_modules'] - 1)
            modules.append(HighResolutionModule(layer_config['num_branches'], block, layer_config['num_blocks'],
                                                num_inchannels, layer_config['num_channels'],
                                                layer_config['fuse_method'], reset))
            num_inchannels = modules[-1].get_num_inchannels()
        return nn.Sequential(*modules), num_inchannels

    def init_weights(self):
        for m in self.modules():
            if isinstance(m, nn.Conv2d):
                nn.init.normal_(m.weight, std=0.001)
                if m.bias is not None:
                    nn.init.constant_(m.bias, 0)
            elif isinstance(m, nn.BatchNorm2d):
                nn.init.constant_(m.weight, 1)
                nn.init.constant_(m.bias, 0)

    def load_weights(self, pretrained=''):
        pretrained = osp.expandvars(pretrained)
        if osp.isfile(pretrained):
            sd = torch.load(pretrained, map_location=torch.device('cpu'))
            need = {k: v for k, v in sd.items()
                    if k.split('.')[0] in self.pretrained_layers or self.pretrained_layers[0] == '*'}
            self.load_state_dict(need, strict=False)
        elif pretrained:
            raise ValueError('{} is not exist!'.format(pretrained))

    # ------------------------------------------------------------------ compilation to the op program
    def _block_ops(self, g, blk, x):
        if isinstance(blk, BasicBlock):
            if blk.downsample is not None:
                raise ValueError('shapy_b200: BasicBlock with a downsample branch is not on the SHAPY_A path '
                                 '(network_defaults.py:92-132 never creates one)')
            t = g.conv(blk.conv1, blk.bn1, x, relu=True)
            return g.conv(blk.conv2, blk.bn2, t, relu=True, res=x)
        idt = x
        if blk.downsample is not None:
            lane = g.lane
            g.on(lane + 1)                                 # independent of conv1 / conv2: runs beside them
            if isinstance(blk.downsample, nn.Conv2d):      # conv_layers: bare 1x1 conv, no BN (hrnet.py:361-373)
                idt = g.conv(blk.downsample, None, x, relu=False)
            else:
                idt = g.conv(blk.downsample[0], blk.downsample[1], x, relu=False)
            g.on(lane)
        t = g.conv(blk.conv1, blk.bn1, x, relu=True)
        t = g.conv(blk.conv2, blk.bn2, t, relu=True)
        return g.conv(blk.conv3, blk.bn3, t, relu=True, res=idt)

    def _module_ops(self, g, mod, xs):
        # branch i runs in lane i: the branches of a module are independent (reference hrnet.py:175-181)
        xs = list(xs)
        for i in range(mod.num_branches):
            g.on(i)
            for blk in mod.branches[i]:
                xs[i] = self._block_ops(g, blk, xs[i])
        if mod.num_branches == 1:
            g.on(0)
            return xs
        # fuse stage: the (i, j) conv chains are independent of each other (hrnet.py:184-191); they are dealt to the lanes
        # longest first onto the least loaded lane (cost ~ MACs + a fixed launch term), the sum of output i runs in lane i
        nout = len(mod.fuse_layers)
        terms = [[None] * mod.num_branches for _ in range(nout)]
        chains = []
        for i in range(nout):
            for j in range(mod.num_branches):
                if j == i:
                    terms[i][j] = (xs[j], 0)
                    continue
                fl = mod.fuse_layers[i][j]
                seqs = [fl] if j > i else list(fl)
                cost, div = 0.0, g.tensors[xs[j]]['div']
                for seq in seqs:
                    c = seq[0]
                    div *= c.stride[0]
                    cost += c.in_channels * c.out_channels * c.kernel_size[0] ** 2 / float(div * div) + 2e3
                chains.append((cost, i, j, seqs))
        load = [0.0] * N_LANES
        for cost, i, j, seqs in sorted(chains, key=lambda c: -c[0]):
            lane = min(range(N_LANES), key=lambda l: load[l])
            load[lane] += cost
            g.on(lane)
            t = xs[j]
            for k, seq in enumerate(seqs):
                t = g.conv(seq[0], seq[1], t, relu=(j < i and k != len(seqs) - 1))
            terms[i][j] = (t, j - i if j > i else 0)
        outs = []
        for i in range(nout):
            g.on(i)
            outs.append(g.fuse(terms[i], relu=True))
        g.on(0)
        return outs

    def build_program(self):
        """Returns (convs, ops, slots, feat_slot, layer_slots): the flat op program of this network."""
        g = _Graph()
        x = g.conv(self.conv1, self.bn1, -1, relu=True)
        x = g.conv(self.conv2, self.bn2, x, relu=True)
        for blk in self.layer1:
            x = self._block_ops(g, blk, x)

        def transition(layers, ys, nprev):
            xs = []
            for i, tl in enumerate(layers):
                g.on(i)
                if tl is None:
                    xs.append(ys[i])
                else:
                    src = ys[i] if i < nprev else ys[-1]
                    if isinstance(tl[0], nn.Conv2d):          # Sequential(conv, bn, relu)
                        xs.append(g.conv(tl[0], tl[1], src, relu=True))
                    else:                                       # Sequential of Sequential(conv, bn, relu)
                        t = src
                        for seq in tl:
                            t = g.conv(seq[0], seq[1], t, relu=True)
                        xs.append(t)
            g.on(0)
            return xs
        ys = transition(self.transition1, [x], 1)
        for mod in self.stage2:
            ys = self._module_ops(g, mod, ys)
        ys = transition(self.transition2, ys, 2)
        for mod in self.stage3:
            ys = self._module_ops(g, mod, ys)
        ys = transition(self.transition3, ys, 3)
        for mod in self.stage4:
            ys = self._module_ops(g, mod, ys)
        for t in ys:
            g.keep.add(t)
        cat = g.tensor(4 * 384, 32)

        def subsample(seq, t, coff):
            n = len(seq) // 3
            for i in range(n):
                last = i == n - 1
                t = g.conv(seq[3 * i], seq[3 * i + 1], t, relu=True, out=cat if last else None,
                           out_coff=coff if last else 0)
            return t
        g.on(0)
        subsample(self.subsample_4, ys[0], 0)
        g.on(1)
        subsample(self.subsample_3, ys[1], 384)
        g.on(2)
        subsample(self.subsample_2, ys[2], 768)
        # x1 = y_list[3] is concatenated as is: copy through a 1-input fuse (no ReLU) into the slice
        g.on(3)
        g.ops.append(dict(kind=OP_FUSE, out_slot=cat, out_coff=1152, relu=0, fuse_in=[ys[3]], fuse_shift=[0], lane=g.lane))
        g.on(0)
        f = cat
        for blk in self.conv_layers:
            f = self._block_ops(g, blk, f)
        g.keep.add(f)
        g.pool(f)
        ops, slots, phys = g.finalize()
        layer_slots = {f'layer{i + 1}': phys[t] for i, t in enumerate(ys)}
        return g.convs, ops, slots, phys[f], layer_slots

    def _compile(self, device):
        convs, ops, slots, feat_slot, layer_slots = self.build_program()
        plan = _ops.HrnetPlan(convs, ops, slots, feat_slot, 2048, int(self.precision_mode), int(self.engine), device)
        return plan, layer_slots

    # ------------------------------------------------------------------ plan cache
    def invalidate(self):
        """Drop the compiled plan (call after editing parameters in place)."""
        self._plan, self._plan_key = None, None

    def _apply(self, fn, *args, **kwargs):          # .to() / .cuda() / .float() / .half()
        self.invalidate()
        return super()._apply(fn, *args, **kwargs)

    def load_state_dict(self, *args, **kwargs):
        self.invalidate()
        return super().load_state_dict(*args, **kwargs)

    def _load_from_state_dict(self, *args, **kwargs):   # reached when a parent module loads a checkpoint
        self.invalidate()
        return super()._load_from_state_dict(*args, **kwargs)

    def plan(self, device):
        key = (str(device), int(self.precision_mode), int(self.engine))
        if self._plan is None or self._plan_key != key:
            self._plan, self._layer_slots = self._compile(device)
            self._plan_key = key
        return self._plan

    def __deepcopy__(self, memo):
        import copy
        plan, key = self._plan, self._plan_key
        self._plan, self._plan_key = None, None
        try:
            cls = self.__class__
            new = cls.__new__(cls)
            memo[id(self)] = new
            for k, v in self.__dict__.items():
                new.__dict__[k] = copy.deepcopy(v, memo)
        finally:
            self._plan, self._plan_key = plan, key
        return new

    def forward(self, x):
        if self.training:
            raise RuntimeError('shapy_b200 HighResolutionNet is inference-only: call .eval() first')
        if not (torch.is_tensor(x) and x.is_cuda):
            raise RuntimeError('shapy_b200 HighResolutionNet: input must be a CUDA tensor (there is no CPU path)')
        plan = self.plan(x.device)
        feats = plan.forward(x)
        return _Outputs(plan, self._layer_slots, feats)
