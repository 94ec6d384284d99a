"""The Planning head (stp3/models/planning_model.py) with the reference's module tree, eval mode on sm_90a.

forward() runs the reference's eval-mode call (planning_model.py:89-150) in four stages:
    reduce_channel      four Bottlenecks on the wgmma convolution kernel: cam_front -> h0 (B, G), NCHW flatten
    stp3_plan_maps      drivable probability, dangerous area and lane-divider cost per BEV cell
    stp3_plan_cost      Cost_Function.forward: cost_fc (B, N), cost_fo (B, N, T)
    stp3_plan_refine    argmin over the command's window of candidates, then T GRUCell steps and the MLP decoder
The command becomes a window (first candidate, count) per sample instead of the reference's three stacked copies of
the chosen third: the argmin over the stacked copies is the argmin over the third.  Nothing is read back to the host.
Training (Planning.loss and its gradients) is not built.
"""
import torch
import torch.nn as nn

from .. import dense, ops
from ..cost import Cost_Function
from ..layers._packing import PackedModule
from ..layers.convolutions import Bottleneck

PLANNING_EVAL_ONLY = ("the planning head is eval-only on sm_90a: its loss and gradients are not implemented -- call "
                      ".eval()")


def reduced_hw(h: int, w: int):
    """Map size after the three downsampling Bottlenecks (each ceil(/2): an odd edge is padded, the 3x3 has stride 2)."""
    for _ in range(3):
        h, w = (h + 1) // 2, (w + 1) // 2
    return h, w


class Planning(PackedModule):
    def __init__(self, cfg, feature_channel, gru_input_size=6, gru_state_size=256):
        super().__init__()
        self.cost_function = Cost_Function(cfg)
        self.sample_num = cfg.PLANNING.SAMPLE_NUM
        self.commands = cfg.PLANNING.COMMAND
        assert self.sample_num % 3 == 0
        self.num = int(self.sample_num / 3)
        if gru_input_size != 6:
            raise NotImplementedError(f"Planning: gru_input_size = {gru_input_size}; the GRU input is the previous "
                                      "output, the selected point and the target point (6 values)")
        if gru_state_size % 32 != 0 or not 32 <= gru_state_size <= 512:
            raise NotImplementedError(f"Planning: gru_state_size = {gru_state_size}; stp3_plan_refine takes a multiple "
                                      "of 32 up to 512")
        ds = cfg.MODEL.ENCODER.DOWNSAMPLE
        hf, wf = cfg.IMAGE.FINAL_DIM[0] // ds, cfg.IMAGE.FINAL_DIM[1] // ds
        h, w = reduced_hw(hf, wf)
        if int(feature_channel / 8) * h * w != gru_state_size:
            raise ValueError(f"Planning: the reduced front-camera features have {int(feature_channel / 8)} x {h} x {w} = "
                             f"{int(feature_channel / 8) * h * w} values but the GRU state has {gru_state_size} (the "
                             "reference would fail at its first GRU step)")
        self.feature_hw = (hf, wf)

        self.reduce_channel = nn.Sequential(
            Bottleneck(feature_channel, feature_channel, downsample=True),
            Bottleneck(feature_channel, int(feature_channel / 2), downsample=True),
            Bottleneck(int(feature_channel / 2), int(feature_channel / 2), downsample=True),
            Bottleneck(int(feature_channel / 2), int(feature_channel / 8))
        )
        self.GRU = nn.GRUCell(gru_input_size, gru_state_size)
        self.decoder = nn.Sequential(
            nn.Linear(gru_state_size, gru_state_size),
            nn.ReLU(inplace=True),
            nn.Linear(gru_state_size, 2)
        )

    def _pack(self):
        f = lambda t: t.detach().float().contiguous()
        return {"w_ih": f(self.GRU.weight_ih), "b_ih": f(self.GRU.bias_ih), "w_hh_t": f(self.GRU.weight_hh.t()),
                "b_hh": f(self.GRU.bias_hh), "w1_t": f(self.decoder[0].weight.t()), "b1": f(self.decoder[0].bias),
                "w2": f(self.decoder[2].weight), "b2": f(self.decoder[2].bias)}

    def _require_eval(self):
        if any(m.training for m in self.modules()):
            raise NotImplementedError(f"Planning: {PLANNING_EVAL_ONLY}")

    def windows(self, commands, B: int, N: int, device):
        """Per-sample candidate window (first, count): LEFT, FORWARD, RIGHT take their third of the N candidates,
        anything else all of them.  Returns the host copy (pinned) and the device copy (non-blocking)."""
        if len(commands) != B:
            raise ValueError(f"{len(commands)} commands for a batch of {B}")
        if N != self.sample_num:
            raise ValueError(f"trajs holds {N} candidates per sample, PLANNING.SAMPLE_NUM is {self.sample_num}")
        k = self.num
        third = {'LEFT': (0, k), 'FORWARD': (k, k), 'RIGHT': (2 * k, N - 2 * k)}
        host = torch.tensor([third.get(c, (0, N)) for c in commands], dtype=torch.int32).pin_memory()
        return host, host.to(device, non_blocking=True)

    def reduce(self, cam_front: torch.Tensor) -> torch.Tensor:
        """cam_front (B, C, Hf, Wf) fp32 -> h0 (B, G): the four Bottlenecks, flattened in (C, H, W) order."""
        if cam_front.ndim != 4 or tuple(cam_front.shape[2:]) != self.feature_hw:
            raise ValueError(f"cam_front: expected (B, C, {self.feature_hw[0]}, {self.feature_hw[1]}), got "
                             f"{tuple(cam_front.shape)}")
        x = dense.from_f32(cam_front.unsqueeze(1))
        for m in self.reduce_channel:
            x = m.forward_hl(x)
        return dense.to_f32(x).reshape(cam_front.shape[0], -1)

    @staticmethod
    def split_hd_map(hd_map):
        if hd_map.shape[1] == 2:
            return hd_map[:, 0:1], hd_map[:, 1:2]
        if hd_map.shape[1] == 4:
            return hd_map[:, 0:2], hd_map[:, 2:4]
        raise NotImplementedError(f"hd_map with {hd_map.shape[1]} channels: 2 (raw lane / drivable) or 4 (logits)")

    def _refine(self, h0, trajs, windows, cost_fc, cost_fo, target_points, n_hd):
        B, N, T, c = trajs.shape
        d = self.cost_function.desc(B, N, T, n_hd, c, G=self.GRU.hidden_size)
        return ops.plan_refine(d, windows[0], windows[1], trajs, cost_fc, cost_fo, h0, target_points, **self.packed())

    def select(self, trajs, cost_volume, semantic_pred, lane_divider, drivable_area, target_points, k=1):
        """The cheapest of all N candidates (planning_model.py:47-64), lowest index on ties: (B, T, 3)."""
        if k != 1:
            raise NotImplementedError("Planning.select: k = 1 only (the reference's only use)")
        self._require_eval()
        B, N, T, _ = trajs.shape
        fc, fo = self.cost_function(cost_volume, trajs, semantic_pred, lane_divider, drivable_area, target_points)
        win = self.windows([None] * B, B, N, trajs.device)
        h0 = torch.zeros((B, self.GRU.hidden_size), dtype=torch.float32, device=trajs.device)
        _, sel = self._refine(h0, trajs, win, fc, fo, target_points, lane_divider.shape[1])
        return trajs[torch.arange(B, device=trajs.device), sel.long()]

    def forward(self, cam_front, trajs, gt_trajs, cost_volume, semantic_pred, hd_map, commands, target_points):
        """cam_front (B, C, Hf, Wf), trajs (B, N, T, 3), gt_trajs (unused in eval, may be None), cost_volume
        (B, T, H, W), semantic_pred (B, T, H, W) bool, hd_map (B, 2 or 4, H, W), commands (B strings), target_points
        (B, 2) -> (0, output_traj (B, T, 3))."""
        self._require_eval()
        B, N, T, _ = trajs.shape
        lane, drivable = self.split_hd_map(hd_map)
        win = self.windows(commands, B, N, trajs.device)
        h0 = self.reduce(cam_front)
        target_points = target_points.to(dtype=h0.dtype)
        fc, fo = self.cost_function(cost_volume, trajs, semantic_pred, lane, drivable, target_points)
        out, _ = self._refine(h0, trajs, win, fc, fo, target_points, lane.shape[1])
        return 0, out
