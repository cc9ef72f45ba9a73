"""Parameter inventory of the DD3D configurations (DLA-34, the DLA-X networks and every VoVNetV2-eSE variant), keyed by the reference's state_dict names.

The names/shapes follow what ``DD3D(cfg).state_dict()`` yields in the reference
(tridet/modeling/dd3d/core.py:19-55; DLA tridet/modeling/feature_extractor/dla.py:24-441; VoVNetV2-eSE
tridet/modeling/feature_extractor/vovnet.py:19-143,188-336; FPN + top blocks dla.py:537-561, vovnet.py:411-454;
heads fcos2d.py:55-108, fcos3d.py:81-139).  tests/test_cpu_oracle.py::test_inventory_and_oracle_vs_live_reference checks this inventory against the
reference's own state_dict when /root/reference is present.
"""
import math
from collections import OrderedDict

# kind tags: "conv" (weight, fan-in init), "bias", "bn_w", "bn_b", "bn_mean", "bn_var", "nbt", "gn_w", "gn_b", "scalar",
# "buffer"


def _conv(specs, name, cout, cin, k, bias=False, role="relu"):
    specs[name + ".weight"] = ((cout, cin, k, k), "conv:" + role)
    if bias:
        specs[name + ".bias"] = ((cout, ), "bias:" + role)


def _bn(specs, name, c, frozen):
    specs[name + ".weight"] = ((c, ), "bn_w")
    specs[name + ".bias"] = ((c, ), "bn_b")
    specs[name + ".running_mean"] = ((c, ), "bn_mean")
    specs[name + ".running_var"] = ((c, ), "bn_var")
    if not frozen:
        specs[name + ".num_batches_tracked"] = ((), "nbt")


def _norm(specs, name, c, norm):
    """get_norm(norm, c) as `name` (ref_standin.get_norm / detectron2): BatchNorm2d ("BN", "SyncBN") has
    num_batches_tracked, FrozenBatchNorm2d does not, GroupNorm(32, c) has an affine only; "" adds nothing.  Any other
    string raises KeyError like get_norm's dict lookup."""
    kind = {"BN": "bn", "SyncBN": "bn", "FrozenBN": "frozen", "GN": "gn", "": None}[norm]
    if kind == "gn" and c % 32:  # nn.GroupNorm(32, c)
        raise ValueError(f"num_channels ({c}) must be divisible by num_groups (32)")
    if kind == "gn":
        specs[name + ".weight"] = ((c, ), "gn_w")
        specs[name + ".bias"] = ((c, ), "gn_b")
    elif kind is not None:
        _bn(specs, name, c, frozen=kind == "frozen")


def _conv_bn(specs, name, cout, cin, k, role="relu", norm="FrozenBN"):
    """DLA-34 Conv2d(bias=norm == "") -> get_norm(norm) (dla.py:33,44,154,230,277,337)."""
    _conv(specs, name, cout, cin, k, bias=norm == "", role=role)
    _norm(specs, name + ".norm", cout, norm)


# The reference's DLA_NAME_TO_BUILDER networks the engine builds (dla.py:358-441), by arch key: (FE.BACKBONE.NAME, levels,
# channels, BottleneckX blocks, residual_root, cardinality).  DLA-X-102-64 is dla102x2, which sets BottleneckX.cardinality = 64
# (dla.py:411).  The engine has its own copy (csrc/engine.cu kDlaSpecs); tests/test_dla_x.py pins both against the reference.
DLA_SPECS = {
    "dla34": ("DLA-34", (1, 1, 1, 2, 2, 1), (16, 32, 64, 128, 256, 512), False, False, 0),
    "dla_x_46_c": ("DLA-X-46-C", (1, 1, 1, 2, 2, 1), (16, 32, 64, 64, 128, 256), True, False, 32),
    "dla_x_60_c": ("DLA-X-60-C", (1, 1, 1, 2, 3, 1), (16, 32, 64, 64, 128, 256), True, False, 32),
    "dla_x_60": ("DLA-X-60", (1, 1, 1, 2, 3, 1), (16, 32, 128, 256, 512, 1024), True, False, 32),
    "dla_x_102": ("DLA-X-102", (1, 1, 1, 3, 4, 1), (16, 32, 128, 256, 512, 1024), True, True, 32),
    "dla_x_102_64": ("DLA-X-102-64", (1, 1, 1, 3, 4, 1), (16, 32, 128, 256, 512, 1024), True, True, 64),
}
DLA_KEYS = {spec[0]: key for key, spec in DLA_SPECS.items()}  # FE.BACKBONE.NAME -> arch key


def _dla_block(specs, p, cin, cout, norm, cardinality):
    """BasicBlock (dla.py:24-62), or BottleneckX (dla.py:104-143) when cardinality > 0: 1x1 -> grouped 3x3 -> 1x1 with
    bottleneck width cout * cardinality / 32 and conv2.weight (width, width / cardinality, 3, 3)."""
    if not cardinality:
        _conv_bn(specs, f"{p}.conv1", cout, cin, 3, norm=norm)
        _conv_bn(specs, f"{p}.conv2", cout, cout, 3, role="linear", norm=norm)
        return
    width = cout * cardinality // 32
    _conv_bn(specs, f"{p}.conv1", width, cin, 1, norm=norm)
    _conv_bn(specs, f"{p}.conv2", width, width // cardinality, 3, norm=norm)
    _conv_bn(specs, f"{p}.conv3", cout, width, 1, role="linear", norm=norm)


def _dla_tree(specs, p, levels, in_ch, out_ch, level_root, root_dim=0, norm="FrozenBN", cardinality=0):
    """Tree (dla.py:170-247) in module registration order: tree1, tree2, root, project (only where tree1 is a block)."""
    if root_dim == 0:
        root_dim = 2 * out_ch
    if level_root:
        root_dim += in_ch
    if levels == 1:
        _dla_block(specs, f"{p}.tree1", in_ch, out_ch, norm, cardinality)
        _dla_block(specs, f"{p}.tree2", out_ch, out_ch, norm, cardinality)
        _conv_bn(specs, f"{p}.root.conv", out_ch, root_dim, 1, norm=norm)
        if in_ch != out_ch:
            _conv_bn(specs, f"{p}.project", out_ch, in_ch, 1, role="linear", norm=norm)
    else:
        _dla_tree(specs, p + ".tree1", levels - 1, in_ch, out_ch, False, norm=norm, cardinality=cardinality)
        _dla_tree(specs, p + ".tree2", levels - 1, out_ch, out_ch, False, root_dim=root_dim + out_ch, norm=norm,
                  cardinality=cardinality)


def _dla(specs, arch, norm):
    p = "backbone.bottom_up"
    _, levels, ch, bottleneck_x, _, cardinality = DLA_SPECS[arch]
    card = cardinality if bottleneck_x else 0
    _conv_bn(specs, p + ".base_layer", ch[0], 3, 7, norm=norm)
    _conv_bn(specs, p + ".level0.0", ch[0], ch[0], 3, norm=norm)
    _conv_bn(specs, p + ".level1.0", ch[1], ch[0], 3, norm=norm)
    _dla_tree(specs, p + ".level2", levels[2], ch[1], ch[2], False, norm=norm, cardinality=card)
    for lvl in (3, 4, 5):
        _dla_tree(specs, p + f".level{lvl}", levels[lvl], ch[lvl - 1], ch[lvl], True, norm=norm, cardinality=card)
    return {f"level{lvl}": ch[lvl] for lvl in range(6)}  # channels of every output (dla.py:309-312)


V99_STAGE_CONV_CH = [128, 160, 192, 224]
V99_STAGE_OUT_CH = [256, 512, 768, 1024]
V99_BLOCKS = [1, 3, 9, 3]

# The reference's VoVNet _STAGE_SPECS (vovnet.py:19-97), by arch key: (FE.BACKBONE.NAME, stem, stage_conv_ch, stage_out_ch,
# layer_per_block, block_per_stage, dw).  The engine has its own copy (csrc/engine.cu kVovSpecs); tests/test_vovnet_family.py
# pins both against the reference.
VOVNET_SPECS = {
    "v2_19_slim_dw": ("V-19-slim-dw-eSE", (64, 64, 64), (64, 80, 96, 112), (112, 256, 384, 512), 3, (1, 1, 1, 1), True),
    "v2_19_dw": ("V-19-dw-eSE", (64, 64, 64), (128, 160, 192, 224), (256, 512, 768, 1024), 3, (1, 1, 1, 1), True),
    "v2_19_slim": ("V-19-slim-eSE", (64, 64, 128), (64, 80, 96, 112), (112, 256, 384, 512), 3, (1, 1, 1, 1), False),
    "v2_19": ("V-19-eSE", (64, 64, 128), (128, 160, 192, 224), (256, 512, 768, 1024), 3, (1, 1, 1, 1), False),
    "v2_39": ("V-39-eSE", (64, 64, 128), (128, 160, 192, 224), (256, 512, 768, 1024), 5, (1, 1, 2, 2), False),
    "v2_57": ("V-57-eSE", (64, 64, 128), (128, 160, 192, 224), (256, 512, 768, 1024), 5, (1, 1, 4, 3), False),
    "v2_99": ("V-99-eSE", (64, 64, 128), tuple(V99_STAGE_CONV_CH), tuple(V99_STAGE_OUT_CH), 5, tuple(V99_BLOCKS), False),
}
VOVNET_KEYS = {spec[0]: key for key, spec in VOVNET_SPECS.items()}  # FE.BACKBONE.NAME -> arch key
ARCH_KEYS = ("dla34", ) + tuple(VOVNET_SPECS) + tuple(k for k in DLA_SPECS if k != "dla34")


def _vov_conv3x3(specs, n, cout, cin, dw, norm):
    """conv3x3 (vovnet.py:124-143) or dw_conv3x3 (vovnet.py:100-121; the reference builds it only with cin == cout)."""
    if dw:
        specs[f"{n}/dw_conv3x3.weight"] = ((cout, 1, 3, 3), "conv:dw")
        _conv(specs, f"{n}/pw_conv1x1", cout, cin, 1)
        _norm(specs, f"{n}/pw_norm", cout, norm)
    else:
        _conv(specs, f"{n}/conv", cout, cin, 3)
        _norm(specs, f"{n}/norm", cout, norm)


def _vovnet(specs, arch, norm):
    """The VoVNet convs never have a bias; every one is followed by get_norm(norm) (vovnet.py:100-159,286-287)."""
    p = "backbone.bottom_up"
    _, stem, stage_ch, out_ch, nl, blocks, dw = VOVNET_SPECS[arch]
    _conv(specs, f"{p}.stem.stem_1/conv", stem[0], 3, 3)
    _norm(specs, f"{p}.stem.stem_1/norm", stem[0], norm)
    _vov_conv3x3(specs, f"{p}.stem.stem_2", stem[1], stem[0], dw, norm)
    _vov_conv3x3(specs, f"{p}.stem.stem_3", stem[2], stem[1], dw, norm)
    in_ch = stem[2]
    for si, (sc, oc, nb) in enumerate(zip(stage_ch, out_ch, blocks), start=2):
        for b in range(nb):
            name = f"OSA{si}_{b + 1}"
            q = f"{p}.stage{si}.{name}"
            cin = in_ch
            if dw and in_ch != sc:  # conv_reduction (vovnet.py:200-205)
                r = f"{q}.conv_reduction.{name}_reduction_0"
                _conv(specs, f"{r}/conv", sc, in_ch, 1)
                _norm(specs, f"{r}/norm", sc, norm)
                cin = sc
            for i in range(nl):
                _vov_conv3x3(specs, f"{q}.layers.{i}.{name}_{i}", sc, cin, dw, norm)
                cin = sc
            _conv(specs, f"{q}.concat.{name}_concat/conv", oc, in_ch + nl * sc, 1)
            _norm(specs, f"{q}.concat.{name}_concat/norm", oc, norm)
            _conv(specs, f"{q}.ese.fc", oc, oc, 1, bias=True, role="ese")
            in_ch = oc
    return dict(stem=stem[2], **{f"stage{si}": oc for si, oc in enumerate(out_ch, start=2)})


def param_specs(cfg):
    """OrderedDict name -> (shape, kind) in the reference's state_dict ORDER-INDEPENDENT naming."""
    specs = OrderedDict()
    specs["pixel_mean"] = ((3, 1, 1), "buffer")
    specs["pixel_std"] = ((3, 1, 1), "buffer")
    arch = arch_of(cfg)
    norm = backbone_norm(cfg)
    feats = _dla(specs, arch, norm) if arch in DLA_SPECS else _vovnet(specs, arch, norm)
    fpn_norm = cfg.FE.FPN.NORM  # detectron2 FPN: bias only without a norm; one norm per conv
    F = fpn_channels(cfg)  # the FPN's width is every head's width too (fcos2d.py:43-45, fcos3d.py:70-72)
    for name, stride in fpn_inputs(cfg):  # registered in FE.FPN.IN_FEATURES order, named by log2 stride
        st = int(math.log2(stride))
        for conv, cin, k in ((f"backbone.fpn_lateral{st}", feats[name], 1), (f"backbone.fpn_output{st}", F, 3)):
            _conv(specs, conv, F, cin, k, bias=fpn_norm == "", role="linear")
            _norm(specs, conv + ".norm", F, fpn_norm)
    _conv(specs, "backbone.top_block.p6", F, F, 3, bias=True, role="linear")
    if arch in DLA_SPECS:
        _conv(specs, "backbone.top_block.p7", F, F, 3, bias=True, role="linear")

    C = cfg.DD3D.NUM_CLASSES
    L = len(in_feature_levels(cfg))  # num_levels = len(in_features): fcos2d.py:36, fcos3d.py:60
    ND = len(cfg.DD3D.FCOS3D.MEAN_DEPTH_PER_LEVEL)  # scales_depth / offsets_depth: one per entry (fcos3d.py:136-139)
    f2, f3 = cfg.DD3D.FCOS2D, cfg.DD3D.FCOS3D
    box3d_on = bool(cfg.MODEL.BOX3D_ON)  # core.py:34-40: no FCOS3D head at all when off
    # fcos2d.py:46-91, fcos3d.py:75-112: NUM_*_CONVS x Conv2d(bias = no norm, norm); BN / FrozenBN one per level
    # (ModuleListDial), any other norm one shared by the levels
    towers = [("fcos2d_head.cls_tower", f2.NUM_CLS_CONVS, f2.NORM), ("fcos2d_head.box2d_tower", f2.NUM_BOX_CONVS, f2.NORM)]
    if box3d_on:
        towers.append(("fcos3d_head.box3d_tower", f3.NUM_CONVS, f3.NORM))
    for tower, depth, norm in towers:
        _norm({}, "", 32, norm)  # KeyError for an unknown NORM even at depth 0
        for i in range(depth):
            _conv(specs, f"{tower}.{i}", F, F, 3, bias=norm == "")
            if norm in ("BN", "FrozenBN"):
                for l in range(L):
                    _norm(specs, f"{tower}.{i}.norm.{l}", F, norm)
            else:
                _norm(specs, f"{tower}.{i}.norm", F, norm)
    _conv(specs, "fcos2d_head.cls_logits", C, F, 3, bias=True, role="cls_logits")
    _conv(specs, "fcos2d_head.box2d_reg", 4, F, 3, bias=True, role="box2d_reg")
    _conv(specs, "fcos2d_head.centerness", 1, F, 3, bias=True, role="centerness")
    if f2.USE_SCALE:  # fcos2d.py:100-108
        for l in range(L):
            specs[f"fcos2d_head.scales_box2d_reg.{l}.scale"] = ((1, ), "scalar:box2d")
    if box3d_on:
        C3 = 1 if f3.CLASS_AGNOSTIC_BOX3D else C          # fcos3d.py:103
        NL = L if f3.PER_LEVEL_PREDICTORS else 1           # fcos3d.py:104
        specs["fcos3d_head.mean_depth_per_level"] = ((ND, ), "buffer")
        specs["fcos3d_head.std_depth_per_level"] = ((ND, ), "buffer")
        for name, mult, role, bias in (("quat", 4, "quat", True), ("ctr", 2, "ctr", True),
                                       ("depth", 1, "depth", not f3.USE_SCALE),  # fcos3d.py:116
                                       ("size", 3, "size", True), ("conf", 1, "conf", True)):
            for li in range(NL):
                _conv(specs, f"fcos3d_head.box3d_{name}.{li}", mult * C3, F, 3, bias=bias, role=role)
        if f3.USE_SCALE:  # fcos3d.py:128-139
            for l in range(max(L, ND)):
                if l < L:
                    specs[f"fcos3d_head.scales_proj_ctr.{l}.scale"] = ((1, ), "scalar:ctr")
                    specs[f"fcos3d_head.scales_size.{l}.scale"] = ((1, ), "scalar:one")
                    specs[f"fcos3d_head.scales_conf.{l}.scale"] = ((1, ), "scalar:one")
                if l < ND:
                    specs[f"fcos3d_head.scales_depth.{l}.scale"] = ((1, ), "scalar:depth")
                    specs[f"fcos3d_head.offsets_depth.{l}.bias"] = ((1, ), "scalar:depth_offset")
    if is_nuscenes_arch(cfg):  # nuscenes_dd3d.py:311-312 (appended last: the synthetic generator stream of the rest is unchanged)
        _conv(specs, "attr_logits", MAX_NUM_ATTRIBUTES, F, 3, bias=True, role="attr")
        _conv(specs, "speed", 1, F, 3, bias=True, role="speed")
    return specs


MAX_NUM_ATTRIBUTES = 3  # tridet/data/datasets/nuscenes/build.py:77

# FE.FPN.OUT_CHANNELS the engine builds (dd3d_set_fpn_channels): every multiple of 64 from 64 to 512
FPN_WIDTHS = tuple(range(64, 513, 64))


def fpn_channels(cfg):
    """FE.FPN.OUT_CHANNELS (configs/feature_extractors/d2_fpn.yaml:5; the reference's FPN builders read it, dla.py:546-557,
    vovnet.py:438-450): the width of the FPN laterals, outputs and top block and of every FCOS head conv."""
    return int(cfg.FE.FPN.OUT_CHANNELS)


def check_fpn_channels(cfg):
    """NotImplementedError for an FPN width the reference builds and the engine does not.  Call it after param_specs, which
    raises the reference's own errors first (GN on a width that 32 does not divide: nn.GroupNorm's ValueError)."""
    c = fpn_channels(cfg)
    if c not in FPN_WIDTHS:
        raise NotImplementedError(f"FE.FPN.OUT_CHANNELS = {c} is not supported: the engine builds "
                                  + ", ".join(str(w) for w in FPN_WIDTHS))
    return c


def is_nuscenes_arch(cfg):
    """MODEL.META_ARCHITECTURE names the reference class ("DD3D" / "NuscenesDD3D", configs/meta_arch/dd3d.yaml:12,
    configs/experiments/dd3d_nusc_*.yaml:9) or its registered B200 mirror ("DD3DB200" / "NuscenesDD3DB200")."""
    name = cfg.MODEL.META_ARCHITECTURE
    if name not in ("DD3D", "NuscenesDD3D", "DD3DB200", "NuscenesDD3DB200"):
        raise KeyError("No object named '{}' found in 'META_ARCH' registry!".format(name))
    return name.startswith("NuscenesDD3D")


def arch_of(cfg):
    """Arch key of FE.BUILDER + FE.BACKBONE.NAME: a key of DLA_SPECS or of VOVNET_SPECS."""
    b = cfg.FE.BUILDER
    if b == "build_fcos_dla_fpn_backbone_p67":
        name = cfg.FE.BACKBONE.NAME
        if name not in DLA_KEYS:  # dla.py also builds DLA-46-C, DLA-60, DLA-102, DLA-169: plain Bottleneck blocks
            raise NotImplementedError(f"DLA variant {name!r} is not supported: the engine builds "
                                      + ", ".join(DLA_KEYS))
        return DLA_KEYS[name]
    if b == "build_fcos_vovnet_fpn_backbone_p6":
        return VOVNET_KEYS[cfg.FE.BACKBONE.NAME]  # KeyError for an unknown name, like _STAGE_SPECS[cfg.NAME]
    raise KeyError("No object named '{}' found in 'BACKBONE' registry!".format(b))


def backbone_norm(cfg):
    """FE.BACKBONE.NORM, with the errors the reference raises for the combinations it cannot build or run: an unknown string
    (KeyError, get_norm's lookup), GN on channel counts that 32 does not divide (ValueError from nn.GroupNorm: DLA-34's 16, the
    slim VoVNets' 112; raised by _norm while the inventory is built) and a VoVNet without a norm.  The reference raises the
    last one only at its first forward, where nn.Sequential calls the None norm (vovnet.py:119,139,159); the mirror raises it
    at construction."""
    norm = cfg.FE.BACKBONE.NORM
    _norm({}, "", 32, norm)  # KeyError for an unknown NORM
    if norm == "" and arch_of(cfg) not in DLA_SPECS:
        raise TypeError("'NoneType' object is not callable")
    return norm


# Stride of every backbone output the reference names: DLA level<k> is 2**k (dla.py:309-312); the VoVNet stem and stage2 are 4,
# each later stage doubles it (vovnet.py:306-333)
DLA_OUTPUT_STRIDES = {f"level{k}": 2**k for k in range(6)}
VOVNET_OUTPUT_STRIDES = {"stem": 4, "stage2": 4, "stage3": 8, "stage4": 16, "stage5": 32}
# The FPN inputs without a configured FE.FPN.IN_FEATURES list (configs/feature_extractors/{dla34,v2_99}_fpn.yaml)
DEFAULT_FPN_INPUTS = {True: ["level3", "level4", "level5"], False: ["stage2", "stage3", "stage4", "stage5"]}


def fpn_inputs(cfg):
    """FE.FPN.IN_FEATURES as [(backbone output, stride)], with the errors the reference raises while it builds the backbone
    and the FPN: the DLA's assert on an output that is not one of its children and KeyError for base_layer (dla.py:300-315),
    KeyError for a VoVNet output it does not have (VoVNet.output_shape), KeyError for an FPN input the backbone does not
    return (``input_shapes[f]``), and detectron2's AssertionErrors for an empty list and for strides that do not double
    from one input to the next (FPN.__init__, _assert_strides_are_log2_contiguous)."""
    dla = arch_of(cfg) in DLA_SPECS
    out = cfg.FE.BACKBONE.OUT_FEATURES
    if dla:
        out = ["level5"] if out is None else list(out)
        assert len(out)
        children = ["base_layer"] + list(DLA_OUTPUT_STRIDES)
        for f in out:
            assert f in children, "Available children: {}".format(", ".join(children))
        shapes = {f: DLA_OUTPUT_STRIDES[f] for f in out}
    else:
        shapes = {f: VOVNET_OUTPUT_STRIDES[f] for f in out}
    in_features = list(cfg.FE.FPN.IN_FEATURES)
    assert in_features, in_features
    strides = [shapes[f] for f in in_features]
    for i, stride in enumerate(strides[1:], 1):
        assert stride == 2 * strides[i - 1], "Strides {} {} are not log2 contiguous".format(stride, strides[i - 1])
    return list(zip(in_features, strides))


def fpn_output_names(cfg):
    """The FPN's outputs in order (backbone.output_shape()): p<log2 stride> of every FPN input, then the top block's p6 and p7
    for the DLA p67 builder (dla.py:536-561) or p6 for the VoVNet p6 builder (vovnet.py:428-454).  The defaults give p3..p7 and
    p2..p6."""
    stages = [int(math.log2(s)) for _, s in fpn_inputs(cfg)]
    top = 2 if arch_of(cfg) in DLA_SPECS else 1
    return [f"p{s}" for s in stages] + [f"p{stages[-1] + k}" for k in range(1, top + 1)]


def check_fpn_inputs(cfg):
    """The errors of an FE.FPN.IN_FEATURES list that builds in the reference but cannot run: the top block reads
    ``results[self._out_features.index("p5")]`` at the first forward, ValueError without a p5 output and IndexError when p5 is
    a top-block output; then NotImplementedError for what the engine does not build: inputs below stride 4 (DLA level0 /
    level1, which its fused front end never stores) and more than DD3D_NUM_LEVELS (5) head levels, the bound of the decode
    and of the NMS shared memory at PRE_NMS_TOPK.  Call it after param_specs, which raises the construction errors."""
    inputs = fpn_inputs(cfg)
    idx = fpn_output_names(cfg).index("p5")
    if idx >= len(inputs):
        raise IndexError("list index out of range")
    low = [f for f, s in inputs if s < 4]
    if low:
        raise NotImplementedError(f"FE.FPN.IN_FEATURES {low} below stride 4 are not supported: the engine builds the FPN on "
                                  "DLA level2..level5 and VoVNet stem / stage2..stage5")
    n = len(in_feature_levels(cfg))
    if n > 5:
        raise NotImplementedError(f"{n} head levels are not supported: the engine runs at most 5 (set DD3D.IN_FEATURES to at "
                                  f"most 5 of {fpn_output_names(cfg)})")


def in_feature_levels(cfg):
    """DD3D.IN_FEATURES as FPN output indices in head order: `cfg.DD3D.IN_FEATURES or list(backbone_output_shape)`
    (core.py:25-26).  An unknown name raises KeyError like the reference's `backbone_output_shape[f]`; a repeated level, which
    the reference builds but has no use, raises NotImplementedError."""
    names = fpn_output_names(cfg)
    dd3d = cfg.DD3D
    sel = dd3d.get("IN_FEATURES") if hasattr(dd3d, "get") else getattr(dd3d, "IN_FEATURES", None)
    sel = list(sel or names)
    for f in sel:
        if f not in names:
            raise KeyError(f)
    for f in sel:
        if sel.count(f) > 1:
            raise NotImplementedError(f"DD3D.IN_FEATURES lists {f!r} {sel.count(f)} times: the engine runs each FPN "
                                      "level at most once")
    return [names.index(f) for f in sel]


def level_strides(cfg):
    """Strides of the head levels, in DD3D.IN_FEATURES order (compute_locations, core.py:166-174)."""
    strides = [2**int(name[1:]) for name in fpn_output_names(cfg)]
    return [strides[i] for i in in_feature_levels(cfg)]


def size_divisibility(cfg):
    return 128 if arch_of(cfg) in DLA_SPECS else 64
