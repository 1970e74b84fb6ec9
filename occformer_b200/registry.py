"""Registry surface of the drop-in boundary.

The reference registers its modules in mmcv registries under fixed names (``NECKS``,
``BACKBONES``, ``HEADS``; e.g. ``@BACKBONES.register_module() class OccupancyEncoder``,
projects/mmdet3d_plugin/occformer/backbones/occnet.py:11) and the configs instantiate them by
``type='<name>'`` (projects/configs/occformer_nusc/occformer_nusc_r50_256x704.py:79-190).

When mmcv / mmdet / mmdet3d are importable our classes are registered into *their* registries
(``force=True`` so that importing this package after the reference plugin swaps the hot-path modules
in place and the unchanged configs build the H100 versions).  When they are not (this image), a
minimal local registry with the same ``register_module`` / ``build`` surface is used.

The image encoder's ``ResNet`` and ``SECONDFPN`` are the exception: general mmdet / mmdet3d names, registered in the
local registries only (``upstream=False``).  The ``OccupancyFormer`` detector resolves those names to this package's
classes for the submodules it builds; a config built outside it opts in as INTEGRATION.md shows.
"""


class Registry:
    def __init__(self, name):
        self.name = name
        self._module_dict = {}

    def get(self, key):
        return self._module_dict.get(key)

    def register_module(self, name=None, force=False, module=None):
        def _reg(cls):
            key = name or cls.__name__
            if key in self._module_dict and not force and self._module_dict[key] is not cls:
                raise KeyError(f"{key} is already registered in {self.name}")
            self._module_dict[key] = cls
            return cls

        if module is not None:
            return _reg(module)
        return _reg

    def build(self, cfg, default_args=None):
        args = dict(cfg)
        if default_args:
            for k, v in default_args.items():
                args.setdefault(k, v)
        t = args.pop("type")
        cls = self.get(t) if isinstance(t, str) else t
        if cls is None:
            raise KeyError(f"{t} is not in the {self.name} registry")
        return cls(**args)


class _Mirror:
    """Registers into the local registry and, when present, into the upstream mmcv registries."""

    def __init__(self, name, upstream_names):
        self.local = Registry(name)
        self.upstreams = []
        for modname, attr in upstream_names:
            try:
                mod = __import__(modname, fromlist=[attr])
                self.upstreams.append(getattr(mod, attr))
            except Exception:
                pass

    def register_module(self, name=None, force=True, module=None, upstream=True):
        """upstream=False registers in the local registry only: for a class whose name is a general mmdet / mmdet3d one
        (ResNet, SECONDFPN) that must not replace the upstream class for other models in the same process; configs reach
        it through the local registry or with the class itself as ``type``."""
        def _reg(cls):
            self.local.register_module(name=name, force=True)(cls)
            for up in self.upstreams if upstream else ():
                try:
                    up.register_module(name=name, force=True)(cls)
                except Exception:
                    pass
            return cls

        if module is not None:
            return _reg(module)
        return _reg

    def get(self, key):
        return self.local.get(key)

    def build(self, cfg, default_args=None):
        return self.local.build(cfg, default_args)


NECKS = _Mirror("neck", [("mmdet3d.models.builder", "NECKS"), ("mmdet.models.builder", "NECKS")])
BACKBONES = _Mirror("backbone", [("mmdet3d.models.builder", "BACKBONES"), ("mmdet.models.builder", "BACKBONES")])
DETECTORS = _Mirror("detector", [("mmdet.models.builder", "DETECTORS"), ("mmdet3d.models.builder", "DETECTORS")])
HEADS = _Mirror("head", [("mmdet.models.builder", "HEADS"), ("mmdet3d.models.builder", "HEADS")])
# mmcv 1.4.0 keeps these two in mmcv.cnn.bricks.registry (re-exported by mmcv.cnn.bricks.transformer); the reference
# registers SinePositionalEncoding3D / MultiScaleDeformableAttention3D there
# (mask2former/positional_encodings/positional_encoding.py:11-12, necks/multi_scale_deform_attn_3d.py:83-84)
POSITIONAL_ENCODING = _Mirror("position encoding", [("mmcv.cnn.bricks.registry", "POSITIONAL_ENCODING"),
                                                    ("mmcv.cnn.bricks.transformer", "POSITIONAL_ENCODING")])
ATTENTION = _Mirror("attention", [("mmcv.cnn.bricks.registry", "ATTENTION"), ("mmcv.cnn.bricks.transformer", "ATTENTION")])
# loader transforms (mmdet 2.x keeps the registry in mmdet.datasets.builder, where the reference registers its loaders,
# P/datasets/pipelines/loading_nusc_occ.py:9,13)
PIPELINES = _Mirror("pipeline", [("mmdet.datasets.builder", "PIPELINES")])
