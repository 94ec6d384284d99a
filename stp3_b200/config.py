"""Attribute-style configuration with the reference's key names and defaults (stp3/config.py:32-162) for the keys the
perception hot path reads.  fvcore/yacs are not needed: `get_cfg()` returns a nested attribute dict; the reference's
YAML overrides (e.g. stp3/configs/nuscenes/Perception.yml) can be applied with `merge(dict)`."""
import copy


class CfgNode(dict):
    def __getattr__(self, k):
        try:
            return self[k]
        except KeyError as e:
            raise AttributeError(k) from e

    def __setattr__(self, k, v):
        self[k] = v

    def merge(self, other):
        for k, v in other.items():
            if isinstance(v, dict) and isinstance(self.get(k), dict):
                self[k].merge(v)
            else:
                self[k] = CfgNode.wrap(v)
        return self

    @staticmethod
    def wrap(v):
        if isinstance(v, dict) and not isinstance(v, CfgNode):
            return CfgNode({k: CfgNode.wrap(x) for k, x in v.items()})
        return v

    def convert_to_dict(self):
        return {k: (v.convert_to_dict() if isinstance(v, CfgNode) else v) for k, v in self.items()}


_DEFAULTS = {
    "TIME_RECEPTIVE_FIELD": 3,
    "N_FUTURE_FRAMES": 4,
    "IMAGE": {"FINAL_DIM": (224, 480), "NAMES": ['CAM_FRONT_LEFT', 'CAM_FRONT', 'CAM_FRONT_RIGHT', 'CAM_BACK_LEFT',
                                                  'CAM_BACK', 'CAM_BACK_RIGHT']},
    "LIFT": {"X_BOUND": [-50.0, 50.0, 0.5], "Y_BOUND": [-50.0, 50.0, 0.5], "Z_BOUND": [-10.0, 10.0, 20.0],
             "D_BOUND": [2.0, 50.0, 1.0], "GT_DEPTH": False, "DISCOUNT": 0.5},
    "MODEL": {
        "ENCODER": {"DOWNSAMPLE": 8, "NAME": 'efficientnet-b4', "OUT_CHANNELS": 64, "USE_DEPTH_DISTRIBUTION": True},
        "TEMPORAL_MODEL": {"NAME": 'temporal_block', "START_OUT_CHANNELS": 64, "EXTRA_IN_CHANNELS": 0,
                           "INBETWEEN_LAYERS": 0, "PYRAMID_POOLING": True, "INPUT_EGOPOSE": True},
        "DISTRIBUTION": {"LATENT_DIM": 32, "MIN_LOG_SIGMA": -5.0, "MAX_LOG_SIGMA": 5.0},
        "FUTURE_PRED": {"N_GRU_BLOCKS": 2, "N_RES_LAYERS": 1, "MIXTURE": True},
        "BN_MOMENTUM": 0.1,
    },
    "SEMANTIC_SEG": {"VEHICLE": {"WEIGHTS": [1.0, 2.0]},
                     "PEDESTRIAN": {"ENABLED": True, "WEIGHTS": [1.0, 10.0]},
                     "HDMAP": {"ENABLED": True, "ELEMENTS": ['lane_divider', 'drivable_area']}},
    "INSTANCE_SEG": {"ENABLED": True},
    "INSTANCE_FLOW": {"ENABLED": True},
    "PROBABILISTIC": {"ENABLED": True, "METHOD": 'GAUSSIAN'},
    "PLANNING": {"ENABLED": True, "GRU_STATE_SIZE": 256, "SAMPLE_NUM": 600, "COMMAND": ['LEFT', 'FORWARD', 'RIGHT']},
    "EGO": {"WIDTH": 1.85, "HEIGHT": 4.084},
    "COST_FUNCTION": {"SAFETY": 0.1, "LAMBDA": 1., "HEADWAY": 1., "LRDIVIDER": 10., "COMFORT": 0.1, "PROGRESS": 0.5,
                      "VOLUME": 100.},
}

# stp3/configs/nuscenes/Perception.yml
PERCEPTION_OVERRIDES = {
    "TIME_RECEPTIVE_FIELD": 3, "N_FUTURE_FRAMES": 0,
    "MODEL": {"ENCODER": {"NAME": 'efficientnet-b4', "USE_DEPTH_DISTRIBUTION": True},
              "TEMPORAL_MODEL": {"NAME": 'temporal_block', "INPUT_EGOPOSE": True}, "BN_MOMENTUM": 0.05},
    "SEMANTIC_SEG": {"PEDESTRIAN": {"ENABLED": True}, "HDMAP": {"ENABLED": True}},
    "INSTANCE_SEG": {"ENABLED": False}, "INSTANCE_FLOW": {"ENABLED": False},
    "PROBABILISTIC": {"ENABLED": False}, "PLANNING": {"ENABLED": False},
}

# stp3/configs/nuscenes/Prediction.yml (apply with get_cfg(PREDICTION_OVERRIDES, perception=False))
PREDICTION_OVERRIDES = {
    "TIME_RECEPTIVE_FIELD": 3, "N_FUTURE_FRAMES": 4,
    "LIFT": {"GT_DEPTH": False},
    "MODEL": {"ENCODER": {"NAME": 'efficientnet-b4', "USE_DEPTH_DISTRIBUTION": True},
              "TEMPORAL_MODEL": {"NAME": 'temporal_block', "INPUT_EGOPOSE": True}, "BN_MOMENTUM": 0.05},
    "SEMANTIC_SEG": {"PEDESTRIAN": {"ENABLED": False}, "HDMAP": {"ENABLED": False}},
    "INSTANCE_FLOW": {"ENABLED": True},
    "PROBABILISTIC": {"ENABLED": True, "METHOD": 'GAUSSIAN'}, "PLANNING": {"ENABLED": False},
}

# stp3/configs/nuscenes/Planning.yml (apply with get_cfg(PLANNING_OVERRIDES, perception=False))
PLANNING_OVERRIDES = {
    "TIME_RECEPTIVE_FIELD": 3, "N_FUTURE_FRAMES": 6,
    "LIFT": {"GT_DEPTH": False},
    "MODEL": {"ENCODER": {"NAME": 'efficientnet-b4', "USE_DEPTH_DISTRIBUTION": True},
              "TEMPORAL_MODEL": {"NAME": 'temporal_block', "INPUT_EGOPOSE": True}, "BN_MOMENTUM": 0.05},
    "SEMANTIC_SEG": {"PEDESTRIAN": {"ENABLED": True}, "HDMAP": {"ENABLED": True}},
    "INSTANCE_SEG": {"ENABLED": False}, "INSTANCE_FLOW": {"ENABLED": False},
    "PROBABILISTIC": {"ENABLED": True, "METHOD": 'GAUSSIAN'},
    "PLANNING": {"ENABLED": True, "SAMPLE_NUM": 1800},
    "COST_FUNCTION": {"SAFETY": 1., "HEADWAY": 1., "LRDIVIDER": 10., "COMFORT": 0.1, "PROGRESS": 0.5, "VOLUME": 100.},
}

# stp3/configs/carla/Planning.yml (apply with get_cfg(PLANNING_CARLA_OVERRIDES, perception=False))
PLANNING_CARLA_OVERRIDES = {
    "TIME_RECEPTIVE_FIELD": 3, "N_FUTURE_FRAMES": 4,
    "IMAGE": {"FINAL_DIM": (256, 256)},
    "LIFT": {"X_BOUND": [-20.0, 20.0, 0.2], "Y_BOUND": [-20.0, 20.0, 0.2], "GT_DEPTH": False},
    "EGO": {"WIDTH": 2.12, "HEIGHT": 4.90},
    "MODEL": {"ENCODER": {"NAME": 'efficientnet-b4', "USE_DEPTH_DISTRIBUTION": True},
              "TEMPORAL_MODEL": {"NAME": 'temporal_block', "INPUT_EGOPOSE": True}, "BN_MOMENTUM": 0.05},
    "SEMANTIC_SEG": {"PEDESTRIAN": {"ENABLED": True}, "HDMAP": {"ENABLED": True}},
    "INSTANCE_SEG": {"ENABLED": False}, "INSTANCE_FLOW": {"ENABLED": False},
    "PROBABILISTIC": {"ENABLED": True, "METHOD": 'GAUSSIAN'},
    "PLANNING": {"ENABLED": True, "GRU_STATE_SIZE": 128, "SAMPLE_NUM": 2400},
    "COST_FUNCTION": {"SAFETY": 1., "HEADWAY": 1., "LRDIVIDER": 10., "COMFORT": 1., "PROGRESS": 1., "VOLUME": 100.},
}


def get_cfg(overrides=None, perception=True):
    """Reference defaults (+ the nuScenes perception YAML when perception=True) + overrides.  COST_FUNCTION's values
    become floats, as the reference's get_cfg makes them (config.py:180-181)."""
    cfg = CfgNode.wrap(copy.deepcopy(_DEFAULTS))
    if perception:
        cfg.merge(PERCEPTION_OVERRIDES)
    if overrides:
        cfg.merge(overrides)
    for k in list(cfg.COST_FUNCTION):
        cfg.COST_FUNCTION[k] = float(cfg.COST_FUNCTION[k])
    return cfg
