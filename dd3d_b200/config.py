"""Config tree for the DD3D inference path.

Mirrors the key hierarchy the reference reads by attribute (``cfg.DD3D.FCOS3D...``, ``cfg.FE...``,
``cfg.MODEL...``) so the same object can drive the reference meta-arch and ``DD3DB200``.  Values restate
reference configs: configs/models/dd3d.yaml, configs/meta_arch/dd3d.yaml:12-19,
configs/feature_extractors/{dla34_fpn,v2_99_fpn,d2_fpn}.yaml, configs/train_datasets/{kitti_3d,nuscenes}.yaml
and the experiment deltas configs/experiments/dd3d_kitti_{dla34,v99}.yaml:13-27 (FrozenBN backbone/FPN/FCOS3D,
eval-mode BN in FCOS2D, NMS_THRESH 0.75).
"""
import copy

from .arch import VOVNET_SPECS


class CfgNode(dict):
    """dict with attribute access, like the OmegaConf/yacs nodes the reference uses."""
    def __getattr__(self, name):
        try:
            return self[name]
        except KeyError as e:
            raise AttributeError(name) from e

    def __setattr__(self, name, value):
        self[name] = value

    def __deepcopy__(self, memo):
        return CfgNode({k: copy.deepcopy(v, memo) for k, v in self.items()})


def _to_node(d):
    if isinstance(d, dict):
        return CfgNode({k: _to_node(v) for k, v in d.items()})
    if isinstance(d, (list, tuple)):
        return [_to_node(v) for v in d]
    return d


KITTI_CANONICAL_BOX3D_SIZES = [  # (width, length, height); configs/train_datasets/kitti_3d.yaml:6-16
    [1.61876949, 3.89154523, 1.52969237],
    [0.62806586, 0.82038497, 1.76784787],
    [0.56898187, 1.77149234, 1.7237099],
    [1.9134491, 5.15499603, 2.18998422],
    [2.61168401, 9.22692319, 3.36492722],
    [0.5390196, 1.08098042, 1.28392158],
    [2.36044838, 15.56991038, 3.5289238],
    [1.24489164, 2.51495357, 1.61402478],
]
NUSC_CANONICAL_BOX3D_SIZES = [  # configs/train_datasets/nuscenes.yaml:6-18
    [2.3524184, 0.5062202, 1.0413622],
    [0.61416006, 1.7016163, 1.3054738],
    [2.9139307, 10.725025, 3.2832346],
    [1.9751819, 4.641267, 1.74352],
    [2.772134, 6.565072, 3.2474296],
    [0.7800532, 2.138673, 1.4437162],
    [0.6667362, 0.7181772, 1.7616143],
    [0.40246472, 0.4027083, 1.0084083],
    [3.0059454, 12.8197, 4.1213827],
    [2.4986045, 6.9310856, 2.8382742],
]

_DATASETS = {
    "kitti_3d": dict(
        NUM_CLASSES=5,
        CANONICAL_BOX3D_SIZES=KITTI_CANONICAL_BOX3D_SIZES,
        MEAN_DEPTH_PER_LEVEL=[32.594, 15.178, 8.424, 5.004, 4.662],
        STD_DEPTH_PER_LEVEL=[14.682, 7.139, 4.345, 2.399, 2.587],
    ),
    "nuscenes": dict(
        NUM_CLASSES=10,
        CANONICAL_BOX3D_SIZES=NUSC_CANONICAL_BOX3D_SIZES,
        MEAN_DEPTH_PER_LEVEL=[44.921, 20.252, 11.712, 7.166, 8.548],
        STD_DEPTH_PER_LEVEL=[24.331, 9.833, 6.223, 4.611, 8.275],
    ),
}

_FEATURE_EXTRACTORS = {
    "dla34": dict(
        BUILDER="build_fcos_dla_fpn_backbone_p67",
        BACKBONE=dict(NAME="DLA-34", OUT_FEATURES=["level3", "level4", "level5"], NORM="FrozenBN"),
    ),
    "v2_99": dict(
        BUILDER="build_fcos_vovnet_fpn_backbone_p6",
        BACKBONE=dict(NAME="V-99-eSE", OUT_FEATURES=["stage2", "stage3", "stage4", "stage5"], NORM="FrozenBN"),
    ),
}
# the other VoVNets of vovnet.py:_STAGE_SPECS: same builder and FPN, FE.BACKBONE.NAME picks the variant
for _key, _spec in VOVNET_SPECS.items():
    if _key not in _FEATURE_EXTRACTORS:
        _FEATURE_EXTRACTORS[_key] = copy.deepcopy(_FEATURE_EXTRACTORS["v2_99"])
        _FEATURE_EXTRACTORS[_key]["BACKBONE"]["NAME"] = _spec[0]


def get_cfg(backbone="dla34", dataset="kitti_3d", nms_thresh=0.75, meta_arch="DD3D", act_dtype="bf16"):
    """backbone: "dla34" or a VoVNet key of dd3d_b200.arch.VOVNET_SPECS ("v2_19_slim_dw", "v2_19_dw", "v2_19_slim", "v2_19",
    "v2_39", "v2_57", "v2_99"), which sets FE.BACKBONE.NAME; dataset in {"kitti_3d", "nuscenes"} (head constants only); meta_arch in
    {"DD3D", "NuscenesDD3D"} (configs/experiments/dd3d_nusc_{dla34,v99}.yaml:9,30-36)."""
    ds = _DATASETS[dataset]
    fe = copy.deepcopy(_FEATURE_EXTRACTORS[backbone])
    fe["FPN"] = dict(IN_FEATURES=list(fe["BACKBONE"]["OUT_FEATURES"]), OUT_FEATURES=None, OUT_CHANNELS=256,
                     NORM="FrozenBN", FUSE_TYPE="sum")
    fe["OUT_FEATURES"] = None
    cfg = dict(
        # test-time resize: configs/experiments/dd3d_kitti_{dla34,v99}.yaml:34, dd3d_nusc_{dla34,v99}.yaml:43-44
        INPUT=dict(FORMAT="BGR", AUG_ENABLED=True,
                   RESIZE=dict(MIN_SIZE_TEST=384 if dataset == "kitti_3d" else 896, MAX_SIZE_TEST=100000)),
        MODEL=dict(
            DEVICE="cuda",
            META_ARCHITECTURE=meta_arch,
            PIXEL_MEAN=[103.530, 116.280, 123.675],
            PIXEL_STD=[57.375, 57.120, 58.395],
            CKPT="",
            BOX2D_ON=True,
            BOX3D_ON=True,
            DEPTH_ON=False,
        ),
        FE=fe,
        DD3D=dict(
            IN_FEATURES=None,
            NUM_CLASSES=ds["NUM_CLASSES"],
            FEATURE_LOCATIONS_OFFSET="none",
            SIZES_OF_INTEREST=[64, 128, 256, 512],
            INFERENCE=dict(DO_NMS=True, DO_POSTPROCESS=True, DO_BEV_NMS=False, BEV_NMS_IOU_THRESH=0.3,
                           NUSC_SAMPLE_AGGREGATE=False),
            FCOS2D=dict(
                _VERSION="v2",
                NORM="BN",
                NUM_CLS_CONVS=4,
                NUM_BOX_CONVS=4,
                USE_DEFORMABLE=False,
                USE_SCALE=True,
                BOX2D_SCALE_INIT_FACTOR=1.0,
                LOSS=dict(ALPHA=0.25, GAMMA=2.0, LOC_LOSS_TYPE="giou"),
                INFERENCE=dict(THRESH_WITH_CTR=True, PRE_NMS_THRESH=0.05, PRE_NMS_TOPK=1000, POST_NMS_TOPK=100,
                               NMS_THRESH=nms_thresh),
            ),
            FCOS3D=dict(
                NORM="FrozenBN",
                NUM_CONVS=4,
                USE_DEFORMABLE=False,
                USE_SCALE=True,
                DEPTH_SCALE_INIT_FACTOR=0.3,
                PROJ_CTR_SCALE_INIT_FACTOR=1.0,
                PER_LEVEL_PREDICTORS=False,
                SCALE_DEPTH_BY_FOCAL_LENGTHS=True,
                SCALE_DEPTH_BY_FOCAL_LENGTHS_FACTOR=500.0,
                MEAN_DEPTH_PER_LEVEL=ds["MEAN_DEPTH_PER_LEVEL"],
                STD_DEPTH_PER_LEVEL=ds["STD_DEPTH_PER_LEVEL"],
                MIN_DEPTH=0.1,
                MAX_DEPTH=80.0,
                CANONICAL_BOX3D_SIZES=ds["CANONICAL_BOX3D_SIZES"],
                CLASS_AGNOSTIC_BOX3D=False,
                PREDICT_ALLOCENTRIC_ROT=True,
                PREDICT_DISTANCE=False,
                LOSS=dict(SMOOTH_L1_BETA=0.05, MAX_LOSS_PER_GROUP_DISENT=20.0, CONF_3D_TEMPERATURE=1.0,
                          WEIGHT_BOX3D=2.0, WEIGHT_CONF3D=1.0),
                PREPARE_TARGET=dict(CENTER_SAMPLE=True, POS_RADIUS=1.5),
            ),
        ),
        # engine-side switch (not a reference key): 16-bit storage type of activations / weights, "bf16" | "fp16"
        B200=dict(ACT_DTYPE=act_dtype),
        # test-time augmentation: configs/experiments/dd3d_kitti_{dla34,v99}.yaml:47-53, dd3d_nusc_v99.yaml:57-63
        # IMS_PER_BATCH: dd3d_kitti_*.yaml 80, dd3d_nusc_dla34.yaml 96, dd3d_nusc_v99.yaml 192
        TEST=dict(IMS_PER_BATCH=80 if dataset == "kitti_3d" else (96 if backbone == "dla34" else 192),
                  AUG=dict(ENABLED=True,
                           MIN_SIZES=[320, 384, 448, 512, 576] if dataset == "kitti_3d" else [640, 768, 896, 1024, 1152],
                           MAX_SIZE=100000, FLIP=True)),
    )
    if meta_arch == "NuscenesDD3D":  # configs/experiments/dd3d_nusc_{dla34,v99}.yaml:30-36,69-71
        cfg["DD3D"]["NUSC"] = dict(LOSS=dict(WEIGHT_ATTR=0.2, WEIGHT_SPEED=0.2),
                                   INFERENCE=dict(NUM_IMAGES_PER_SAMPLE=6, MAX_NUM_DETS_PER_SAMPLE=500))
        cfg["DATALOADER"] = dict(TEST=dict(NUM_IMAGES_PER_GROUP=6))
    return _to_node(cfg)
