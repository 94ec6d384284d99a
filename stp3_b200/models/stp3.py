"""STP3 perception model with the reference's constructor / forward surface (stp3/models/stp3.py:15-184) for the
perception configuration (N_FUTURE_FRAMES = 0, PLANNING disabled): Encoder -> lift-splat -> TemporalModel -> Decoder,
every stage on hand-written sm_90a kernels behind the C ABI.

Device data flow of forward():
    Encoder heads (wgmma)  -> feature / depth-logit tensors
    stp3_lift_splat_fwd      -> BEV grid directly as channels-last bf16 hi/lo planes + per-(b,t,c) spatial sums
    TemporalModel (wgmma)  -> ego-motion channels and pooling branches enter as per-image biases
    Decoder (wgmma)        -> fp32 logits in the reference's (B,S,k,X,Y) layout
With N_FUTURE_FRAMES > 0 (the Prediction configurations, eval mode only) the present distribution and the future
prediction run between the temporal model and the decoder, and the decoder sees the present and future frames
(DESIGN.md §3.16).  With PLANNING.ENABLED (the Planning configurations, eval mode only) the model also builds the
Planning head (models/planning_model.py, DESIGN.md §3.17) and every forward entry point returns `cam_front`, the
context features of camera 1 at the last present frame, for model.planning.
"""
import torch
import torch.nn as nn

from .. import dense, ops
from ..layers.convolutions import PREDICT_EVAL_ONLY
from ..utils import geometry as G
from .decoder import Decoder
from .distributions import DistributionModule
from .future_prediction import FuturePrediction
from .planning_model import Planning
from .encoder import Encoder
from .temporal_model import TemporalModel, TemporalModelIdentity


class STP3(nn.Module):
    def __init__(self, cfg, backbone=None):
        super().__init__()
        self.cfg = cfg
        res, start, dim = G.calculate_birds_eye_view_parameters(cfg.LIFT.X_BOUND, cfg.LIFT.Y_BOUND, cfg.LIFT.Z_BOUND)
        self.bev_resolution = nn.Parameter(res, requires_grad=False)
        self.bev_start_position = nn.Parameter(start, requires_grad=False)
        self.bev_dimension = nn.Parameter(dim, requires_grad=False)
        self.encoder_downsample = cfg.MODEL.ENCODER.DOWNSAMPLE
        self.encoder_out_channels = cfg.MODEL.ENCODER.OUT_CHANNELS
        self.frustum = self.create_frustum()
        self.depth_channels = self.frustum.shape[0]
        self.discount = cfg.LIFT.DISCOUNT
        if cfg.TIME_RECEPTIVE_FIELD == 1:
            assert cfg.MODEL.TEMPORAL_MODEL.NAME == 'identity'
        self.receptive_field = cfg.TIME_RECEPTIVE_FIELD
        self.n_future = cfg.N_FUTURE_FRAMES
        if cfg.PLANNING.ENABLED:
            if self.n_future == 0:
                raise NotImplementedError("PLANNING.ENABLED with N_FUTURE_FRAMES = 0: the planner scores its candidates on "
                                          "the predicted future frames, and there are none")
            if not (cfg.SEMANTIC_SEG.HDMAP.ENABLED and cfg.SEMANTIC_SEG.PEDESTRIAN.ENABLED):
                raise NotImplementedError("PLANNING.ENABLED needs SEMANTIC_SEG.HDMAP and SEMANTIC_SEG.PEDESTRIAN: the eval-"
                                          "mode planner reads the model's own hdmap logits and vehicle / pedestrian "
                                          "occupancy, as both reference Planning.yml files configure it")
        if self.n_future > 0:
            if cfg.MODEL.TEMPORAL_MODEL.NAME == 'identity':
                raise NotImplementedError("N_FUTURE_FRAMES > 0 with the identity temporal model: the prediction stage is "
                                          "wired behind the temporal_block model only")
            if cfg.PROBABILISTIC.ENABLED and cfg.PROBABILISTIC.METHOD != 'GAUSSIAN':
                raise NotImplementedError(f"PROBABILISTIC.METHOD = {cfg.PROBABILISTIC.METHOD}: only the GAUSSIAN present "
                                          "distribution is built on sm_90a (BERNOULLI / MIXGAUSSIAN are not)")
        if self.encoder_out_channels % 64 != 0:
            raise NotImplementedError(f"MODEL.ENCODER.OUT_CHANNELS = {self.encoder_out_channels}: the tensor-core layers carry "
                                      "channels in blocks of 64 (the reference's configs use 64; the stress configuration 128)")
        if cfg.MODEL.TEMPORAL_MODEL.NAME == 'temporal_block' and cfg.MODEL.TEMPORAL_MODEL.INBETWEEN_LAYERS != 0:
            raise NotImplementedError("MODEL.TEMPORAL_MODEL.INBETWEEN_LAYERS > 0 (Bottleneck3D, temporal.py:328-372) is not used "
                                      "by any reference config and is not built")
        if cfg.TIME_RECEPTIVE_FIELD > 8:
            raise NotImplementedError("TIME_RECEPTIVE_FIELD > 8: the lift-splat keeps the ego-motion chain of at most 8 frames")
        self.spatial_extent = (cfg.LIFT.X_BOUND[1], cfg.LIFT.Y_BOUND[1])
        self.bev_size = (int(dim[0]), int(dim[1]))

        self.encoder = Encoder(cfg=cfg.MODEL.ENCODER, D=self.depth_channels, backbone=backbone)

        temporal_in = self.encoder_out_channels + (6 if cfg.MODEL.TEMPORAL_MODEL.INPUT_EGOPOSE else 0)
        if cfg.MODEL.TEMPORAL_MODEL.NAME == 'identity':
            self.temporal_model = TemporalModelIdentity(temporal_in, self.receptive_field)
        elif cfg.MODEL.TEMPORAL_MODEL.NAME == 'temporal_block':
            self.temporal_model = TemporalModel(
                temporal_in, self.receptive_field, input_shape=self.bev_size,
                start_out_channels=cfg.MODEL.TEMPORAL_MODEL.START_OUT_CHANNELS,
                extra_in_channels=cfg.MODEL.TEMPORAL_MODEL.EXTRA_IN_CHANNELS,
                n_spatial_layers_between_temporal_layers=cfg.MODEL.TEMPORAL_MODEL.INBETWEEN_LAYERS,
                use_pyramid_pooling=cfg.MODEL.TEMPORAL_MODEL.PYRAMID_POOLING)
            if cfg.MODEL.TEMPORAL_MODEL.INPUT_EGOPOSE and len(self.temporal_model.model) > 0:
                self.temporal_model.model[0].n_const = 6
        else:
            raise NotImplementedError(f'Temporal module {cfg.MODEL.TEMPORAL_MODEL.NAME}.')
        self.future_pred_in_channels = self.temporal_model.out_channels
        self.latent_dim = cfg.MODEL.DISTRIBUTION.LATENT_DIM
        if self.n_future > 0:
            if cfg.PROBABILISTIC.ENABLED:
                self.present_distribution = DistributionModule(self.future_pred_in_channels, self.latent_dim,
                                                               method=cfg.PROBABILISTIC.METHOD)
            self.future_prediction = FuturePrediction(
                in_channels=self.future_pred_in_channels, latent_dim=self.latent_dim, n_future=self.n_future,
                mixture=cfg.MODEL.FUTURE_PRED.MIXTURE, n_gru_blocks=cfg.MODEL.FUTURE_PRED.N_GRU_BLOCKS,
                n_res_layers=cfg.MODEL.FUTURE_PRED.N_RES_LAYERS)

        self.decoder = Decoder(
            in_channels=self.future_pred_in_channels, n_classes=len(cfg.SEMANTIC_SEG.VEHICLE.WEIGHTS),
            n_present=self.receptive_field, n_hdmap=len(cfg.SEMANTIC_SEG.HDMAP.ELEMENTS),
            predict_gate={'perceive_hdmap': cfg.SEMANTIC_SEG.HDMAP.ENABLED,
                          'predict_pedestrian': cfg.SEMANTIC_SEG.PEDESTRIAN.ENABLED,
                          'predict_instance': cfg.INSTANCE_SEG.ENABLED,
                          'predict_future_flow': cfg.INSTANCE_FLOW.ENABLED,
                          'planning': cfg.PLANNING.ENABLED})
        if cfg.PLANNING.ENABLED:
            self.planning = Planning(cfg, self.encoder_out_channels, 6, gru_state_size=cfg.PLANNING.GRU_STATE_SIZE)
        for m in self.modules():
            if isinstance(m, (nn.BatchNorm1d, nn.BatchNorm2d, nn.BatchNorm3d)):
                m.momentum = cfg.MODEL.BN_MOMENTUM
        self._ws = ops.Workspace()
        self.stage_events = None        # bench.py sets this to a list to receive (stage name, CUDA event) marks

    # ------------------------------------------------------------------------------------------------ geometry
    def create_frustum(self):
        """(D, Hf, Wf, 3) grid of (u, v, depth), kept as a parameter for state-dict compatibility (stp3.py:111-130);
        the kernels only use its three 1-D axes."""
        xs, ys, ds = G.frustum_axes(self.cfg.IMAGE.FINAL_DIM, self.encoder_downsample, self.cfg.LIFT.D_BOUND)
        D, Hf, Wf = ds.numel(), ys.numel(), xs.numel()
        fr = torch.stack((xs.view(1, 1, Wf).expand(D, Hf, Wf), ys.view(1, Hf, 1).expand(D, Hf, Wf),
                          ds.view(D, 1, 1).expand(D, Hf, Wf)), -1)
        return nn.Parameter(fr.contiguous(), requires_grad=False)

    def _axes(self):
        fr = self.frustum
        return fr[0, 0, :, 0].contiguous(), fr[0, :, 0, 1].contiguous(), fr[:, 0, 0, 2].contiguous()

    def _bev_host(self):
        """(offset, resolution, dimension) as host values, evaluated once with the reference's fp32 tensor expression."""
        cached = self.__dict__.get("_bev_host_cache")
        if cached is None:
            res, start, dim = (t.detach().cpu() for t in (self.bev_resolution, self.bev_start_position, self.bev_dimension))
            cached = (G.bev_offset(start, res), res, dim)
            self.__dict__["_bev_host_cache"] = cached
        return cached

    def prepare_inputs(self, intrinsics, extrinsics, future_egomotion):
        """Host-side parameters of one batch, computed with the reference's own torch calls (SURVEY.md §7-1): camera
        matrices R.K^-1 | t, ego poses R | t, and the shifted ego-motion vector that replaces the six broadcast
        channels of stp3.py:145-152.  Small CPU tensors (a few hundred floats)."""
        S = self.receptive_field
        intrinsics, extrinsics = intrinsics[:, :S].float().cpu(), extrinsics[:, :S].float().cpu()
        ego = future_egomotion[:, :S].float().cpu().contiguous()
        cam_M, cam_t, ego_R, ego_t = G.lift_matrices(intrinsics, extrinsics, ego)
        const = self._shifted_egomotion(ego).reshape(-1, 6).contiguous()
        return {"cam_M": cam_M, "cam_t": cam_t, "ego_R": ego_R, "ego_t": ego_t, "const": const}

    def projection_to_birds_eye_view(self, feat, depth_logits, intrinsics, extrinsics, future_egomotion,
                                     feat_channels_last=False):
        """(B,S,N,C,Hf,Wf) features [or (B,S,N,Hf,Wf,C) with feat_channels_last] + (B,S,N,D,Hf,Wf) depth logits ->
        (B,S,C,X,Y) fp32, as stp3.py:226-301 (which takes the materialised outer product and geometry instead; both are
        fused away here)."""
        h = self.prepare_inputs(intrinsics, extrinsics, future_egomotion)
        off, res, dim = self._bev_host()
        needs_grad = torch.is_grad_enabled() and (feat.requires_grad or (depth_logits is not None and depth_logits.requires_grad))
        fn = ops.lift_splat_autograd if needs_grad else ops.lift_splat      # training through the lift: SURVEY.md row f2
        return fn(feat, depth_logits, h["cam_M"], h["cam_t"], h["ego_R"], h["ego_t"], *self._axes(), off, res,
                  dim, float(self.discount), feat_channels_last=feat_channels_last,
                  use_depth_distribution=self.cfg.MODEL.ENCODER.USE_DEPTH_DISTRIBUTION, workspace=self._ws)

    # ------------------------------------------------------------------------------------------------ forward
    def forward(self, image, intrinsics, extrinsics, future_egomotion):
        """image (B,T,N,3,H,W), intrinsics (B,T,N,3,3), extrinsics (B,T,N,4,4), future_egomotion (B,T,6) -> dict with
        the reference's keys (stp3.py:132-184)."""
        self._check_predict_eval()
        S = self.receptive_field
        image = image[:, :S].contiguous()
        if self.encoder.native:
            dev = image.device
            h = {k: v.to(dev) for k, v in self.prepare_inputs(intrinsics, extrinsics, future_egomotion).items()}
            return self.forward_images_device(image, **h)
        b, s, n = image.shape[:3]
        r_lo, r_hi = self.encoder.trunk(image.view(b * s * n, *image.shape[3:]))
        r_lo = r_lo.float().contiguous().view(b, s, n, *r_lo.shape[1:])
        r_hi = r_hi.float().contiguous().view(b, s, n, *r_hi.shape[1:])
        return self.forward_trunk_features(r_lo, r_hi, intrinsics, extrinsics, future_egomotion)

    def forward_trunk_features(self, r_lo, r_hi, intrinsics, extrinsics, future_egomotion):
        """forward() entering after the (third-party) EfficientNet trunk: r_lo (B,S,N,c3,H/8,W/8), r_hi
        (B,S,N,c4,H/16,W/16) -- the encoder heads (encoder.py:88-95) run on the wgmma kernels and hand their context
        features to the lift-splat channels-last."""
        self._check_predict_eval()
        S = self.receptive_field
        dev = r_lo.device
        h = {k: v.to(dev) for k, v in self.prepare_inputs(intrinsics, extrinsics, future_egomotion).items()}
        return self.forward_heads_device(r_lo[:, :S].contiguous(), r_hi[:, :S].contiguous(), **h)

    def forward_images_device(self, image, cam_M, cam_t, ego_R, ego_t, const):
        """Device-only from images (B,S,N,3,H,W) fp32 through the native trunk: trunk -> heads -> forward_device
        (capturable in a CUDA graph, GraphedPerception(entry="images"))."""
        b, s, n = image.shape[:3]
        self._check_predict_eval()
        self._check_encoder_train()
        self._mark("start_trunk")
        feat, depth = self.encoder.features_native(image.reshape(b * s * n, *image.shape[3:]), channels_last=True)
        feat = feat.view(b, s, n, *feat.shape[1:])
        depth = depth.view(b, s, n, *depth.shape[1:]) if depth is not None else None
        self._mark("encoder")
        return self.forward_device(feat, depth, cam_M, cam_t, ego_R, ego_t, const, feat_channels_last=True)

    def forward_heads_device(self, r_lo, r_hi, cam_M, cam_t, ego_R, ego_t, const):
        """Device-only: encoder heads -> forward_device (capturable in a CUDA graph)."""
        b, s, n = r_lo.shape[:3]
        self._check_predict_eval()
        self._check_encoder_train()
        self._mark("start_heads")
        feat, depth = self.encoder.heads_f32(r_lo.view(b * s * n, *r_lo.shape[3:]), r_hi.view(b * s * n, *r_hi.shape[3:]),
                                             channels_last=True)
        feat = feat.view(b, s, n, *feat.shape[1:])
        depth = depth.view(b, s, n, *depth.shape[1:]) if depth is not None else None
        self._mark("encoder_heads")
        return self.forward_device(feat, depth, cam_M, cam_t, ego_R, ego_t, const, feat_channels_last=True)

    def forward_features(self, feat, depth_logits, intrinsics, extrinsics, future_egomotion, feat_channels_last=False):
        """Same as forward() but entering after the image encoder: feat (B,S,N,C,Hf,Wf) [or (B,S,N,Hf,Wf,C) with
        feat_channels_last], depth_logits (B,S,N,D,Hf,Wf)."""
        self._check_predict_eval()
        S = self.receptive_field
        dev = feat.device
        h = {k: v.to(dev) for k, v in self.prepare_inputs(intrinsics, extrinsics, future_egomotion).items()}
        feat = feat[:, :S].contiguous()
        depth_logits = depth_logits[:, :S].contiguous() if depth_logits is not None else None
        return self.forward_device(feat, depth_logits, **h, feat_channels_last=feat_channels_last)

    def forward_device(self, feat, depth_logits, cam_M, cam_t, ego_R, ego_t, const, feat_channels_last=False):
        """Device-only part of the forward pass (every argument already on the GPU; no host synchronisation, so the
        whole call can be captured in a CUDA graph -- see GraphedPerception)."""
        B, S = feat.shape[:2]
        dev = feat.device
        X, Y = self.bev_size
        C = self.encoder_out_channels
        off, res, dim = self._bev_host()
        output = {'depth_prediction': depth_logits, 'cam_front': self._cam_front(feat, feat_channels_last)}
        self._check_predict_eval()
        if self._head_training() and not self.decoder.training:
            raise RuntimeError("STP3: temporal_model.final_conv is in train mode but the decoder is in eval mode, so no "
                               "gradient could reach the head -- call model.decoder.train() as well")
        use_ego = self.cfg.MODEL.TEMPORAL_MODEL.INPUT_EGOPOSE
        if isinstance(self.temporal_model, TemporalModel) and self.temporal_model.blocks_training():
            # train-mode TemporalBlocks take fp32 BEV features; through the lift-splat's autograd when feat / depth
            # require grad
            needs_grad = torch.is_grad_enabled() and (feat.requires_grad or
                                                      (depth_logits is not None and depth_logits.requires_grad))
            fn = ops.lift_splat_autograd if needs_grad else ops.lift_splat
            bev = fn(feat, depth_logits, cam_M, cam_t, ego_R, ego_t, *self._axes(), off, res, dim, float(self.discount),
                     feat_channels_last=feat_channels_last, workspace=self._ws,
                     use_depth_distribution=self.cfg.MODEL.ENCODER.USE_DEPTH_DISTRIBUTION)
            states = self.temporal_model(bev, const=const if use_ego else None)
            output.update(self.decoder(states))
            return output

        self._mark("start")
        planes = torch.empty((2, B, S, X, Y, C), dtype=torch.bfloat16, device=dev)
        use_pool = isinstance(self.temporal_model, TemporalModel) and len(self.temporal_model.model) > 0 and \
            self.temporal_model.model[0].use_pyramid_pooling
        r = ops.lift_splat(feat, depth_logits, cam_M, cam_t, ego_R, ego_t, *self._axes(), off, res, dim,
                           float(self.discount), use_depth_distribution=self.cfg.MODEL.ENCODER.USE_DEPTH_DISTRIBUTION,
                           workspace=self._ws, out_hilo=planes, pool_sum=use_pool, feat_channels_last=feat_channels_last)
        sums = r[1].view(B * S, C) if use_pool else None
        x = dense.HL(planes[0], planes[1], C)
        self._mark("lift_splat")

        if isinstance(self.temporal_model, TemporalModelIdentity):
            bev = dense.to_f32(x, 0, C)
            if use_ego:
                bev = torch.cat([bev, const.view(B, S, 6, 1, 1).expand(B, S, 6, X, Y)], dim=2)
            states = dense.from_f32(bev)
        else:
            states = self.temporal_model.forward_hl(x, const=const if use_ego else None, sums=sums)
        self._mark("temporal_model")
        if self.n_future > 0:
            states = self._predict_hl(states)
        # a train-mode head hands over fp32 (B, S, C, X, Y) with a grad_fn, for the train-mode decoder
        output.update(self.decoder(states) if torch.is_tensor(states) else self.decoder.forward_hl(states))
        self._mark("decoder")
        return output

    def _cam_front(self, feat, channels_last=False, cam_front_index=1):
        """stp3.py:209-211,315: the context features of camera 1 at the last present frame, (B, C, Hf, Wf) fp32, when
        planning is on (None otherwise).  feat is (B, S, N, C, Hf, Wf), or (B, S, N, Hf, Wf, C) when channels_last."""
        if not self.cfg.PLANNING.ENABLED:
            return None
        if feat.shape[2] <= cam_front_index:
            raise ValueError(f"planning reads the front camera (index {cam_front_index}) but the rig has {feat.shape[2]} "
                             "camera(s)")
        x = feat[:, -1, cam_front_index]
        return (x.permute(0, 3, 1, 2) if channels_last else x).float().contiguous()

    def _predict_hl(self, states: dense.HL) -> dense.HL:
        """Prediction stage (stp3.py:157-176): present distribution of the last present state (eval: the sample is mu,
        broadcast over the map; zeros without PROBABILISTIC) -> future prediction.  HL (B, S, X, Y, C) present states
        -> HL (B, S + n_future, X, Y, C)."""
        B, S, X, Y, _ = states.hi.shape
        self._mark("start_predict")
        sample = None
        if self.cfg.PROBABILISTIC.ENABLED:
            present = dense.HL.empty(B, 1, X, Y, states.c, states.hi.device, cp=states.hi.shape[-1])
            dense.hl_copy((states, 0, S - 1), present, states.hi.shape[-1], T=1)
            mu_log_sigma = self.present_distribution.forward_hl(present)
            sample = dense.HL.empty(B, 1, X, Y, self.latent_dim, states.hi.device)
            dense.hl_broadcast(mu_log_sigma, sample, self.latent_dim)
        self._mark("distribution")
        y = self.future_prediction.forward_hl(sample, states)
        self._mark("future_prediction")
        return y

    def _check_predict_eval(self):
        """Every entry point refuses a Prediction model with a train-mode module before any work is enqueued."""
        if self.n_future > 0 and any(m.training for m in self.modules()):
            raise NotImplementedError(f"STP3: {PREDICT_EVAL_ONLY}")

    def _head_training(self) -> bool:
        return isinstance(self.temporal_model, TemporalModel) and self.temporal_model.final_conv.training

    def _check_encoder_train(self):
        """Train-mode encoder heads need a train-mode path behind them: only the train-mode TemporalBlocks take the
        lift-splat through autograd, and the head and the decoder carry the gradient to them.  A train-mode native
        trunk needs train-mode heads behind it for the same reason."""
        if not self.encoder.heads_training():
            if self.encoder.trunk_training():
                raise RuntimeError("STP3: the native trunk is in train mode but the encoder heads are in eval mode, so "
                                   "no gradient could reach it -- call model.encoder.train_heads() as well, or "
                                   "model.encoder.backbone.eval()")
            return
        if not isinstance(self.temporal_model, TemporalModel):
            raise RuntimeError("STP3: the encoder heads are in train mode, which needs the temporal_block model (the "
                               "identity temporal model runs the inference forward only) -- call "
                               "model.encoder.train_heads(False)")
        if not (self.temporal_model.blocks_training() and self._head_training() and self.decoder.training):
            raise RuntimeError("STP3: the encoder heads are in train mode but the temporal model or the decoder is in "
                               "eval mode, so no gradient could reach them -- call model.temporal_model.train() and "
                               "model.decoder.train() as well")

    def _blocks_training(self) -> bool:
        return isinstance(self.temporal_model, TemporalModel) and any(b.training for b in self.temporal_model.model)

    def forward_features_frame_sharded(self, feat, depth_logits, intrinsics, extrinsics, future_egomotion, gather="nccl"):
        """Latency mode for a global batch smaller than the number of GPUs (SURVEY.md §8e): the B*S camera frames are
        split across the ranks of the default process group, every rank splats only its frames, ONE all-gather of
        the raw BEV grids follows, and the (cheap, elementwise) discount recurrence, the temporal model and the
        decoder run replicated.  Every rank passes the same full inputs and returns the same outputs.
        gather = "nccl": ncclAllGather of the frames; gather = "peer": the finalize kernel's epilogue stores every frame
        into all ranks' buffers over NVLink itself (symmetric memory, parallel.PeerFrameBuffer) -- compute and collective in
        one kernel, bracketed by two device-side barriers."""
        S = self.receptive_field
        dev = feat.device
        if self.encoder.heads_training():
            raise RuntimeError("frame-sharded forward: the encoder heads are in train mode; the sharded path runs the "
                               "inference forward only -- call model.encoder.train_heads(False)")
        if self.encoder.trunk_training():
            raise RuntimeError("frame-sharded forward: the native trunk is in train mode; the sharded path runs the "
                               "inference forward only -- call model.encoder.backbone.eval()")
        h = {k: v.to(dev) for k, v in self.prepare_inputs(intrinsics, extrinsics, future_egomotion).items()}
        feat = feat[:, :S].contiguous()
        depth_logits = depth_logits[:, :S].contiguous() if depth_logits is not None else None
        return self.forward_device_frame_sharded(feat, depth_logits, **h, gather=gather)

    def forward_device_frame_sharded(self, feat, depth_logits, cam_M, cam_t, ego_R, ego_t, const, gather="peer"):
        """Device-only part of the frame-sharded forward (no host synchronisation): with gather="peer" the whole step --
        splat of this rank's frames with the all-gather in the finalize epilogue, the two device-side barriers, discount,
        temporal model, decoder -- can be captured in ONE CUDA graph (GraphedPerception(entry="sharded"))."""
        from .. import parallel
        if self.n_future > 0:
            raise NotImplementedError("frame-sharded forward with N_FUTURE_FRAMES > 0: the latency mode is wired for the "
                                      "perception configurations only")
        h = {"cam_M": cam_M, "cam_t": cam_t, "ego_R": ego_R, "ego_t": ego_t, "const": const}
        dev = feat.device
        B, S = feat.shape[:2]
        X, Y = self.bev_size
        C = self.encoder_out_channels
        off, res, dim = self._bev_host()
        rank, world = parallel.world()
        f0, fc = parallel.shard_batch(B * S, rank, world)
        if gather == "peer" and world > 1:
            key = (B * S, X, Y, C, str(dev))
            pf = self.__dict__.get("_peer_frames")
            if pf is None or pf[0] != key:
                pf = (key, parallel.PeerFrameBuffer(B * S, X, Y, C, dev))
                self.__dict__["_peer_frames"] = pf
            pf = pf[1]
            pf.barrier()                       # every rank has consumed the buffer's previous contents
            if fc > 0:
                ops.lift_splat_frames(feat, depth_logits, h["cam_M"], h["cam_t"], h["ego_R"], h["ego_t"], *self._axes(),
                                      off, res, dim, f0, fc,
                                      use_depth_distribution=self.cfg.MODEL.ENCODER.USE_DEPTH_DISTRIBUTION,
                                      workspace=self._ws, peer_ptrs=pf.ptrs)
            pf.barrier()                       # every rank's stores have landed
            raw = pf.buf.view(B, S, X, Y, C)
        else:
            if fc > 0:
                raw = ops.lift_splat_frames(feat, depth_logits, h["cam_M"], h["cam_t"], h["ego_R"], h["ego_t"], *self._axes(),
                                            off, res, dim, f0, fc,
                                            use_depth_distribution=self.cfg.MODEL.ENCODER.USE_DEPTH_DISTRIBUTION,
                                            workspace=self._ws)
            else:
                raw = torch.empty((0, X, Y, C), dtype=torch.float32, device=dev)
            raw = parallel.all_gather_frames(raw, B * S).view(B, S, X, Y, C)
        planes = ops.bev_discount(raw, float(self.discount))
        x = dense.HL(planes[0], planes[1], C)
        output = {'depth_prediction': depth_logits, 'cam_front': None}
        use_ego = self.cfg.MODEL.TEMPORAL_MODEL.INPUT_EGOPOSE
        if isinstance(self.temporal_model, TemporalModelIdentity):
            raise NotImplementedError("frame-sharded mode is wired for the temporal_block model")
        if self._blocks_training():
            raise RuntimeError("frame-sharded forward: the TemporalBlocks are in train mode; the sharded path runs the "
                               "inference forward only -- call .eval() on temporal_model.model")
        if self._head_training():
            raise RuntimeError("frame-sharded forward: temporal_model.final_conv is in train mode; the sharded path runs "
                               "the inference forward only -- call .eval() on it")
        states = self.temporal_model.forward_hl(x, const=h["const"] if use_ego else None, sums=None)
        output.update(self.decoder.forward_hl(states))
        return output

    def _mark(self, name):
        if self.stage_events is not None:
            ev = torch.cuda.Event(enable_timing=True)
            ev.record()
            self.stage_events.append((name, ev))

    @staticmethod
    def _shifted_egomotion(future_egomotion):
        """stp3.py:148-151: frame t sees the ego-motion of frame t-1, frame 0 sees zeros."""
        return torch.cat([torch.zeros_like(future_egomotion[:, :1]), future_egomotion[:, :-1]], dim=1).float()

    def calculate_birds_eye_view_features(self, x, intrinsics, extrinsics, future_egomotion):
        """(B,S,N,3,H,W) images -> (bev (B,S,C,X,Y) fp32, depth logits (B,S,N,D,Hf,Wf), cam_front) (stp3.py:303-318);
        cam_front is (B,C,Hf,Wf) with planning on, else None."""
        b, s, n = x.shape[:3]
        feat, depth = self.encoder(x.view(b * s * n, *x.shape[3:]))
        feat = feat.view(b, s, n, *feat.shape[1:])
        depth = depth.view(b, s, n, *depth.shape[1:]) if depth is not None else None
        return (self.projection_to_birds_eye_view(feat, depth, intrinsics, extrinsics, future_egomotion), depth,
                self._cam_front(feat))


class GraphedPerception:
    """STP3.forward_features for a fixed batch size replayed as ONE CUDA graph: the ~70 kernel launches of a step
    (lift-splat, wgmma convolutions, helpers) are captured once -- tensor maps and kernel arguments are baked in, all
    buffers are static -- so a step costs one graph launch instead of ~70 Python/ctypes launches.

        g = GraphedPerception(model, batch)
        out = g(feat, depth_logits, intrinsics, extrinsics, future_egomotion)   # host or device tensors
    The returned tensors are the graph's static output buffers (overwritten by the next call)."""

    def __init__(self, model: STP3, batch: int, n_cameras: int, device=None, entry: str = "lift"):
        """entry "lift": the step enters at the encoder outputs (feat, depth_logits), STP3.forward_features;
        entry "heads": at the trunk endpoints (r_lo, r_hi), STP3.forward_trunk_features (encoder heads included);
        entry "sharded": like "lift" but frame-sharded over the ranks of the default process group (latency mode);
        entry "images": from the camera images (B,S,N,3,H,W) through the native trunk, STP3.forward -- the first two
        arguments of __call__ / stage_inputs are then (image, None)."""
        if model.decoder.training:
            raise RuntimeError("GraphedPerception: the decoder is in train mode (batch statistics, running-statistics "
                               "updates, autograd); a CUDA graph replays the inference forward only -- call .eval()")
        if model._blocks_training():
            raise RuntimeError("GraphedPerception: the TemporalBlocks are in train mode (batch statistics, autograd); a "
                               "CUDA graph replays the inference forward only -- call .eval() on temporal_model.model")
        if model._head_training():
            raise RuntimeError("GraphedPerception: temporal_model.final_conv is in train mode (batch statistics, "
                               "dropout, autograd); a CUDA graph replays the inference forward only -- call .eval()")
        if model.encoder.heads_training():
            raise RuntimeError("GraphedPerception: the encoder heads are in train mode (batch statistics, dropout, "
                               "autograd); a CUDA graph replays the inference forward only -- call "
                               "model.encoder.train_heads(False)")
        if model.encoder.trunk_training():
            raise RuntimeError("GraphedPerception: the native trunk is in train mode (batch statistics, drop-connect, "
                               "autograd); a CUDA graph replays the inference forward only -- call "
                               "model.encoder.backbone.eval()")
        self.model = model
        self.entry = entry
        dev = torch.device(device) if device is not None else next(model.parameters()).device
        S, C, D = model.receptive_field, model.encoder_out_channels, model.depth_channels
        Hf, Wf = model.frustum.shape[1:3]
        N = n_cameras
        f32 = dict(dtype=torch.float32, device=dev)
        if entry in ("lift", "sharded"):
            self.big = ("feat", "depth_logits")
            first = {"feat": torch.zeros((batch, S, N, C, Hf, Wf), **f32),
                     "depth_logits": torch.zeros((batch, S, N, D, Hf, Wf), **f32)}
            # "sharded": the frame-sharded latency mode (all ranks capture and replay in lock-step; the exchange of the BEV
            # frames is the finalize kernel's peer stores, so the graph holds no NCCL node)
            self._fwd = model.forward_device if entry == "lift" else model.forward_device_frame_sharded
        elif entry == "heads":
            enc = model.encoder
            idx = {8: 3, 16: 4}[enc.downsample]
            c_lo, c_hi = enc.reduction_channel[idx], enc.reduction_channel[idx + 1]
            self.big = ("r_lo", "r_hi")
            first = {"r_lo": torch.zeros((batch, S, N, c_lo, Hf, Wf), **f32),
                     "r_hi": torch.zeros((batch, S, N, c_hi, Hf // 2, Wf // 2), **f32)}
            self._fwd = model.forward_heads_device
        elif entry == "images":
            if not model.encoder.native:
                raise ValueError('entry="images" needs the native trunk (Encoder backbone="native")')
            H, W = model.cfg.IMAGE.FINAL_DIM
            self.big = ("image",)
            first = {"image": torch.zeros((batch, S, N, 3, H, W), **f32)}
            self._fwd = model.forward_images_device
        else:
            raise ValueError(entry)
        self.static = {
            **first,
            "cam_M": torch.zeros((batch, S, N, 3, 3), **f32), "cam_t": torch.zeros((batch, S, N, 3), **f32),
            "ego_R": torch.zeros((batch, S, 3, 3), **f32), "ego_t": torch.zeros((batch, S, 3), **f32),
            "const": torch.zeros((batch * S, 6), **f32),
        }
        self.pinned = {k: torch.zeros(v.shape, dtype=torch.float32).pin_memory()
                       for k, v in self.static.items() if k not in self.big}
        self.h2d_done = torch.cuda.Event()      # the pinned staging buffers may be rewritten once this has fired
        self.h2d_done.record(torch.cuda.current_stream(dev))
        with torch.no_grad():
            side = torch.cuda.Stream(device=dev)
            side.wait_stream(torch.cuda.current_stream(dev))
            with torch.cuda.stream(side):
                for _ in range(2):                      # warm-up: weight packing, workspace allocation, lazy init
                    self._fwd(**self.static)
            torch.cuda.current_stream(dev).wait_stream(side)
            torch.cuda.synchronize(dev)
            # the graph bakes in the device pointers of the packed / folded weights: remember which parameter versions
            # they were derived from, and keep the packed tensors alive for as long as the graph exists
            self._packed_modules = [m for m in model.modules() if hasattr(m, "packed") and "_packed_cache" in m.__dict__]
            self._signatures = [m._signature() for m in self._packed_modules]
            self._keepalive = [m.__dict__["_packed_cache"] for m in self._packed_modules]
            self.graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(self.graph):
                self.out = self._fwd(**self.static)
            # ... and the lift-splat workspace it splats into: a later eager call may replace model._ws's buffer by a
            # larger one (another batch, or the deterministic mode's int64 grid), and the graph must not replay into
            # freed memory
            if model._ws.buf is not None:
                self._keepalive.append(model._ws.buf)

    def check_weights_unchanged(self):
        """Raises if a parameter or buffer the captured kernels read was modified (load_state_dict, optimizer step,
        .to()) after the capture: the graph would keep replaying the old packed weights."""
        for m, sig in zip(self._packed_modules, self._signatures):
            if m._signature() != sig:
                raise RuntimeError(f"{type(m).__name__}: parameters changed after the CUDA graph was captured; build a new "
                                   "GraphedPerception (the graph holds the packed weights of the old values)")

    def stage_inputs(self, feat, depth_logits, intrinsics, extrinsics, future_egomotion, stream=None):
        """Host-side calibration math + the (asynchronous) copies into the graph's static input buffers.  The pinned
        staging buffers are reused every call: wait until the previous call's H2D copies have left them."""
        self.check_weights_unchanged()
        host = self.model.prepare_inputs(intrinsics, extrinsics, future_egomotion)
        self.h2d_done.synchronize()
        for k, v in host.items():
            self.pinned[k].copy_(v)
            self.static[k].copy_(self.pinned[k], non_blocking=True)
        self.h2d_done.record(stream if stream is not None else torch.cuda.current_stream(self.static["cam_M"].device))
        S = self.model.receptive_field
        self.static[self.big[0]].copy_(feat[:, :S], non_blocking=True)          # (feat, depth_logits), (r_lo, r_hi), (image,)
        if len(self.big) > 1:
            self.static[self.big[1]].copy_(depth_logits[:, :S], non_blocking=True)

    def __call__(self, feat, depth_logits, intrinsics, extrinsics, future_egomotion):
        """Inputs are consumed asynchronously (pinned host tensors must stay untouched until the step has run); the
        returned tensors are the graph's static output buffers, valid until the next call."""
        self.stage_inputs(feat, depth_logits, intrinsics, extrinsics, future_egomotion)
        self.graph.replay()
        return self.out


class PipelinedPerception:
    """Throughput front-end for host-resident inputs: `depth` GraphedPerception slots, host->device copies of step
    i+1 and device->host copies of step i-1 run on copy streams while step i replays its CUDA graph.

        pipe = PipelinedPerception(model, batch, n_cameras)
        pipe.submit(feat, depth_logits, intrinsics, extrinsics, future_egomotion)      # pinned host tensors
        ...                                                                            # (submit up to `depth` steps)
        out = pipe.collect()        # oldest outstanding step: dict of pinned host tensors (reused every `depth` steps)
    """

    def __init__(self, model: STP3, batch: int, n_cameras: int, depth: int = 2, device=None,
                 keys=("segmentation", "pedestrian", "hdmap"), entry: str = "lift"):
        self.model = model
        dev = torch.device(device) if device is not None else next(model.parameters()).device
        self.dev = dev
        self.slots = [GraphedPerception(model, batch, n_cameras, dev, entry=entry) for _ in range(depth)]
        self.keys = [k for k in keys if self.slots[0].out.get(k) is not None]
        self.host_out = [{k: torch.empty(sl.out[k].shape, dtype=torch.float32).pin_memory() for k in self.keys}
                         for sl in self.slots]
        self.copy_in, self.copy_out = torch.cuda.Stream(device=dev), torch.cuda.Stream(device=dev)
        self.ev_in = [torch.cuda.Event() for _ in self.slots]
        self.ev_done = [torch.cuda.Event() for _ in self.slots]
        self.ev_out = [torch.cuda.Event() for _ in self.slots]
        self.head = self.tail = self.inflight = 0
        self.between_steps = None      # optional callable enqueued on the compute stream before every replay

    def submit(self, feat, depth_logits, intrinsics, extrinsics, future_egomotion):
        assert self.inflight < len(self.slots), "collect() a finished step before submitting another one"
        i = self.head
        sl = self.slots[i]
        compute = torch.cuda.current_stream(self.dev)
        with torch.cuda.stream(self.copy_in):
            self.copy_in.wait_event(self.ev_done[i])          # the slot's previous replay has consumed its inputs
            sl.stage_inputs(feat, depth_logits, intrinsics, extrinsics, future_egomotion, stream=self.copy_in)
            self.ev_in[i].record(self.copy_in)
        compute.wait_event(self.ev_in[i])
        compute.wait_event(self.ev_out[i])                    # the slot's previous outputs have left the device
        if self.between_steps is not None:
            self.between_steps()
        sl.graph.replay()
        self.ev_done[i].record(compute)
        with torch.cuda.stream(self.copy_out):
            self.copy_out.wait_event(self.ev_done[i])
            for k in self.keys:
                self.host_out[i][k].copy_(sl.out[k], non_blocking=True)
            self.ev_out[i].record(self.copy_out)
        self.head = (i + 1) % len(self.slots)
        self.inflight += 1

    def collect(self):
        assert self.inflight > 0
        i = self.tail
        self.ev_out[i].synchronize()
        self.tail = (i + 1) % len(self.slots)
        self.inflight -= 1
        return self.host_out[i]
