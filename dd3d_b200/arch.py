"""Parameter inventory of the DD3D configurations (DLA-34 and every VoVNetV2-eSE variant), keyed by the reference's state_dict names.

The names/shapes follow what ``DD3D(cfg).state_dict()`` yields in the reference
(tridet/modeling/dd3d/core.py:19-55; DLA-34 tridet/modeling/feature_extractor/dla.py:250-361; VoVNetV2-eSE
tridet/modeling/feature_extractor/vovnet.py:19-143,188-336; FPN + top blocks dla.py:537-561, vovnet.py:411-454;
heads fcos2d.py:55-108, fcos3d.py:81-139).  tests/test_cpu_oracle.py::test_inventory_and_oracle_vs_live_reference checks this inventory against the
reference's own state_dict when /root/reference is present.
"""
from collections import OrderedDict

# kind tags: "conv" (weight, fan-in init), "bias", "bn_w", "bn_b", "bn_mean", "bn_var", "nbt", "gn_w", "gn_b", "scalar",
# "buffer"


def _conv(specs, name, cout, cin, k, bias=False, role="relu"):
    specs[name + ".weight"] = ((cout, cin, k, k), "conv:" + role)
    if bias:
        specs[name + ".bias"] = ((cout, ), "bias:" + role)


def _bn(specs, name, c, frozen=True):
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
    if kind == "gn":
        specs[name + ".weight"] = ((c, ), "gn_w")
        specs[name + ".bias"] = ((c, ), "gn_b")
    elif kind is not None:
        _bn(specs, name, c, frozen=kind == "frozen")


def _conv_bn(specs, name, cout, cin, k, role="relu"):
    _conv(specs, name, cout, cin, k, role=role)
    _bn(specs, name + ".norm", cout)


def _dla_tree(specs, p, levels, in_ch, out_ch, level_root, root_dim=0):
    if root_dim == 0:
        root_dim = 2 * out_ch
    if level_root:
        root_dim += in_ch
    if levels == 1:
        for t, cin in (("tree1", in_ch), ("tree2", out_ch)):
            _conv_bn(specs, f"{p}.{t}.conv1", out_ch, cin, 3)
            _conv_bn(specs, f"{p}.{t}.conv2", out_ch, out_ch, 3, role="linear")
        _conv_bn(specs, f"{p}.root.conv", out_ch, root_dim, 1)
        if in_ch != out_ch:
            _conv_bn(specs, f"{p}.project", out_ch, in_ch, 1, role="linear")
    else:
        _dla_tree(specs, p + ".tree1", levels - 1, in_ch, out_ch, False)
        _dla_tree(specs, p + ".tree2", levels - 1, out_ch, out_ch, False, root_dim=root_dim + out_ch)


def _dla34(specs):
    p = "backbone.bottom_up"
    ch = [16, 32, 64, 128, 256, 512]
    levels = [1, 1, 1, 2, 2, 1]
    _conv_bn(specs, p + ".base_layer", ch[0], 3, 7)
    _conv_bn(specs, p + ".level0.0", ch[0], ch[0], 3)
    _conv_bn(specs, p + ".level1.0", ch[1], ch[0], 3)
    _dla_tree(specs, p + ".level2", levels[2], ch[1], ch[2], False)
    for lvl in (3, 4, 5):
        _dla_tree(specs, p + f".level{lvl}", levels[lvl], ch[lvl - 1], ch[lvl], True)
    return {"level3": 128, "level4": 256, "level5": 512}


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
ARCH_KEYS = ("dla34", ) + tuple(VOVNET_SPECS)


def _vov_conv3x3(specs, n, cout, cin, dw):
    """conv3x3 (vovnet.py:124-143) or dw_conv3x3 (vovnet.py:100-121; the reference builds it only with cin == cout)."""
    if dw:
        specs[f"{n}/dw_conv3x3.weight"] = ((cout, 1, 3, 3), "conv:dw")
        _conv(specs, f"{n}/pw_conv1x1", cout, cin, 1)
        _bn(specs, f"{n}/pw_norm", cout)
    else:
        _conv(specs, f"{n}/conv", cout, cin, 3)
        _bn(specs, f"{n}/norm", cout)


def _vovnet(specs, arch):
    p = "backbone.bottom_up"
    _, stem, stage_ch, out_ch, nl, blocks, dw = VOVNET_SPECS[arch]
    _conv(specs, f"{p}.stem.stem_1/conv", stem[0], 3, 3)
    _bn(specs, f"{p}.stem.stem_1/norm", stem[0])
    _vov_conv3x3(specs, f"{p}.stem.stem_2", stem[1], stem[0], dw)
    _vov_conv3x3(specs, f"{p}.stem.stem_3", stem[2], stem[1], dw)
    in_ch = stem[2]
    for si, (sc, oc, nb) in enumerate(zip(stage_ch, out_ch, blocks), start=2):
        for b in range(nb):
            name = f"OSA{si}_{b + 1}"
            q = f"{p}.stage{si}.{name}"
            cin = in_ch
            if dw and in_ch != sc:  # conv_reduction (vovnet.py:200-205)
                r = f"{q}.conv_reduction.{name}_reduction_0"
                _conv(specs, f"{r}/conv", sc, in_ch, 1)
                _bn(specs, f"{r}/norm", sc)
                cin = sc
            for i in range(nl):
                _vov_conv3x3(specs, f"{q}.layers.{i}.{name}_{i}", sc, cin, dw)
                cin = sc
            _conv(specs, f"{q}.concat.{name}_concat/conv", oc, in_ch + nl * sc, 1)
            _bn(specs, f"{q}.concat.{name}_concat/norm", oc)
            _conv(specs, f"{q}.ese.fc", oc, oc, 1, bias=True, role="ese")
            in_ch = oc
    return {f"stage{si}": oc for si, oc in enumerate(out_ch, start=2)}


def param_specs(cfg):
    """OrderedDict name -> (shape, kind) in the reference's state_dict ORDER-INDEPENDENT naming."""
    specs = OrderedDict()
    specs["pixel_mean"] = ((3, 1, 1), "buffer")
    specs["pixel_std"] = ((3, 1, 1), "buffer")
    arch = arch_of(cfg)
    if arch == "dla34":
        feats = _dla34(specs)
        stages = {"level3": 3, "level4": 4, "level5": 5}
    else:
        feats = _vovnet(specs, arch)
        stages = {"stage2": 2, "stage3": 3, "stage4": 4, "stage5": 5}
    fpn_norm = cfg.FE.FPN.NORM  # detectron2 FPN: bias only without a norm; one norm per conv
    for name, ch in feats.items():
        st = stages[name]
        for conv, cin, k in ((f"backbone.fpn_lateral{st}", ch, 1), (f"backbone.fpn_output{st}", 256, 3)):
            _conv(specs, conv, 256, cin, k, bias=fpn_norm == "", role="linear")
            _norm(specs, conv + ".norm", 256, fpn_norm)
    _conv(specs, "backbone.top_block.p6", 256, 256, 3, bias=True, role="linear")
    if arch == "dla34":
        _conv(specs, "backbone.top_block.p7", 256, 256, 3, bias=True, role="linear")

    C = cfg.DD3D.NUM_CLASSES
    L = 5
    f2, f3 = cfg.DD3D.FCOS2D, cfg.DD3D.FCOS3D
    box3d_on = bool(cfg.MODEL.BOX3D_ON)  # core.py:34-40: no FCOS3D head at all when off
    # fcos2d.py:46-91, fcos3d.py:75-112: NUM_*_CONVS x Conv2d(bias = no norm, norm); BN / FrozenBN one per level
    # (ModuleListDial), any other norm one shared by the levels
    towers = [("fcos2d_head.cls_tower", f2.NUM_CLS_CONVS, f2.NORM), ("fcos2d_head.box2d_tower", f2.NUM_BOX_CONVS, f2.NORM)]
    if box3d_on:
        towers.append(("fcos3d_head.box3d_tower", f3.NUM_CONVS, f3.NORM))
    for tower, depth, norm in towers:
        _norm({}, "", 256, norm)  # KeyError for an unknown NORM even at depth 0
        for i in range(depth):
            _conv(specs, f"{tower}.{i}", 256, 256, 3, bias=norm == "")
            if norm in ("BN", "FrozenBN"):
                for l in range(L):
                    _norm(specs, f"{tower}.{i}.norm.{l}", 256, norm)
            else:
                _norm(specs, f"{tower}.{i}.norm", 256, norm)
    _conv(specs, "fcos2d_head.cls_logits", C, 256, 3, bias=True, role="cls_logits")
    _conv(specs, "fcos2d_head.box2d_reg", 4, 256, 3, bias=True, role="box2d_reg")
    _conv(specs, "fcos2d_head.centerness", 1, 256, 3, bias=True, role="centerness")
    if f2.USE_SCALE:  # fcos2d.py:100-108
        for l in range(L):
            specs[f"fcos2d_head.scales_box2d_reg.{l}.scale"] = ((1, ), "scalar:box2d")
    if box3d_on:
        C3 = 1 if f3.CLASS_AGNOSTIC_BOX3D else C          # fcos3d.py:103
        NL = L if f3.PER_LEVEL_PREDICTORS else 1           # fcos3d.py:104
        specs["fcos3d_head.mean_depth_per_level"] = ((L, ), "buffer")
        specs["fcos3d_head.std_depth_per_level"] = ((L, ), "buffer")
        for name, mult, role, bias in (("quat", 4, "quat", True), ("ctr", 2, "ctr", True),
                                       ("depth", 1, "depth", not f3.USE_SCALE),  # fcos3d.py:116
                                       ("size", 3, "size", True), ("conf", 1, "conf", True)):
            for li in range(NL):
                _conv(specs, f"fcos3d_head.box3d_{name}.{li}", mult * C3, 256, 3, bias=bias, role=role)
        if f3.USE_SCALE:  # fcos3d.py:128-139
            for l in range(L):
                specs[f"fcos3d_head.scales_proj_ctr.{l}.scale"] = ((1, ), "scalar:ctr")
                specs[f"fcos3d_head.scales_size.{l}.scale"] = ((1, ), "scalar:one")
                specs[f"fcos3d_head.scales_conf.{l}.scale"] = ((1, ), "scalar:one")
                specs[f"fcos3d_head.scales_depth.{l}.scale"] = ((1, ), "scalar:depth")
                specs[f"fcos3d_head.offsets_depth.{l}.bias"] = ((1, ), "scalar:depth_offset")
    if is_nuscenes_arch(cfg):  # nuscenes_dd3d.py:311-312 (appended last: the synthetic generator stream of the rest is unchanged)
        _conv(specs, "attr_logits", MAX_NUM_ATTRIBUTES, 256, 3, bias=True, role="attr")
        _conv(specs, "speed", 1, 256, 3, bias=True, role="speed")
    return specs


MAX_NUM_ATTRIBUTES = 3  # tridet/data/datasets/nuscenes/build.py:77


def is_nuscenes_arch(cfg):
    """MODEL.META_ARCHITECTURE names the reference class ("DD3D" / "NuscenesDD3D", configs/meta_arch/dd3d.yaml:12,
    configs/experiments/dd3d_nusc_*.yaml:9) or its registered B200 mirror ("DD3DB200" / "NuscenesDD3DB200")."""
    name = cfg.MODEL.META_ARCHITECTURE
    if name not in ("DD3D", "NuscenesDD3D", "DD3DB200", "NuscenesDD3DB200"):
        raise KeyError("No object named '{}' found in 'META_ARCH' registry!".format(name))
    return name.startswith("NuscenesDD3D")


def arch_of(cfg):
    """Arch key of FE.BUILDER + FE.BACKBONE.NAME: "dla34" or a key of VOVNET_SPECS."""
    b = cfg.FE.BUILDER
    if b == "build_fcos_dla_fpn_backbone_p67":
        name = cfg.FE.BACKBONE.NAME
        if name != "DLA-34":  # dla.py builds DLA-46-C, DLA-60, ... too: Bottleneck / BottleneckX blocks the engine lacks
            raise NotImplementedError(f"DLA variant {name!r} is not supported: only DLA-34 is built by the engine")
        return "dla34"
    if b == "build_fcos_vovnet_fpn_backbone_p6":
        return VOVNET_KEYS[cfg.FE.BACKBONE.NAME]  # KeyError for an unknown name, like _STAGE_SPECS[cfg.NAME]
    raise KeyError("No object named '{}' found in 'BACKBONE' registry!".format(b))


def level_strides(cfg):
    return [8, 16, 32, 64, 128] if arch_of(cfg) == "dla34" else [4, 8, 16, 32, 64]


def size_divisibility(cfg):
    return 128 if arch_of(cfg) == "dla34" else 64
