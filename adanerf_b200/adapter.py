"""Drop-in for `TrainConfig.inference` (thomasneff/AdaNeRF src/train_data.py:278-299).

`B200Inference.inference(batch, gradient=False, is_inference=True)` has the reference's signature and return
shape -- `(postprocessed_outs, inference_dicts)` -- so `src/evaluate.py:216-235`, `src/plots.py:51-52,237,353`
and `src/export.py:64` can call it unchanged (INTEGRATION.md shows the two-line patch that installs it on an
existing TrainConfig).  Only the entries those callers read are produced:

    outs[-1][:, :3]                          rgb                                (evaluate.py:228)
    dicts[-1]["AdaptiveSamplePositions"]     samples per ray / K                 (evaluate.py:223-224)
    dicts[1]["OracleWeights"]                raw sampling-net output, thr == 0   (evaluate.py:279-280)

With rayMarchSampler FromClassifiedDepth (sampler=1, the DONeRF baseline) the reference's shading-net dict has neither
AdaptiveSamplePositions (the feature set is not adaptive, features.py:561-563) nor OracleWeights (its losses[0] is the
sampler's transform loss, not NeRFWeightMultiplicationLoss, features.py:503-504), and neither has this one's.
A one-network run (rayMarchSampler LinearlySpacedZNearZFar, sampler=2, plain NeRF) returns `([rgb], [dict])`: one network,
one dict, as TrainConfig.inference of a one-model run does.
    dicts[i]["PostProcessedNetworkOutput"]   = outs[i]                           (util/helper.py:79-130)

A batch of several images (ImagePose [n_images, 3], RayDirectionsSamples [n_images, n_samples, 3]) is rendered in one
views call; every output is then [n_images * n_samples, ...], image-major, as the reference's flattened outputs are.

The batch keys are the reference's DatasetKeyConstants (src/datasets.py:24-38)."""
import torch

from .onnx_weights import PDF_TRANSFORMS
from .renderer import Renderer

# the rayMarchSampler of a one-network (plain NeRF) run, on world and on NDC scenes (src/nerf_raymarch_common.py:261-326)
LINEAR_SAMPLERS = ("LinearlySpacedZNearZFar", "LinearlySpacedZNearZFarNoDepthRange")

# src/datasets.py:29-35 and src/features.py:20-40
KEY_POSE, KEY_ROT, KEY_DIRS = "ImagePose", "ImageRotation", "RayDirectionsSamples"
KEY_POST, KEY_NET_OUT = "PostProcessedNetworkOutput", "NetworkOutputBatch"
KEY_ASP, KEY_ORACLE = "AdaptiveSamplePositions", "OracleWeights"
# FeatureSetKeyConstants (src/features.py:20-40) of the auxiliary tensors RayMarchFromPoses.postprocess stores
KEY_WEIGHTS, KEY_ALPHA, KEY_ZVALS, KEY_DEPTH = "NeRFWeightsOutput", "NeRFAlphaOutput", "NeRFInputFeatureZVals", "NeRFOutputDepth"


class B200Inference:
    """scene: dict (view_cell_center, view_cell_size, depth_range [warped], max_depth, fov) -- the fields
    FeatureSet.initialize reads from DatasetInfo (src/features.py:343-360, :747-767)."""

    def __init__(self, scene, sampling_net, shading_net, threshold, num_samples, device=0, want_oracle_weights=None,
                 want_aux=False, sampler=0, pdf_transform=1):
        """sampler / pdf_transform: the renderer options of the same names (0 = the adaptive sampler; 1 = FromClassifiedDepth
        with transform 1 = sigmoid or 2 = softmax; 2 = LinearlySpacedZNearZFar, plain NeRF: sampling_net is None and
        inference returns one network's outputs; threshold is not used by 1 and 2)."""
        self.renderer = Renderer(scene, device=device, sampling_net=sampling_net, shading_net=shading_net)
        self.threshold = float(threshold)
        self.K = int(num_samples)
        self.sampler = int(sampler)
        if self.sampler:
            self.renderer.set_option("sampler", self.sampler)
        if self.sampler == 1:
            self.renderer.set_option("pdf_transform", int(pdf_transform))
        default_ow = self.threshold == 0.0 and not self.sampler
        self.want_oracle_weights = default_ow if want_oracle_weights is None else bool(want_oracle_weights)
        # plots.render_all_imgs / the depth export read NeRFWeightsOutput, NeRFAlphaOutput, NeRFOutputDepth (src/plots.py:272-306)
        self.want_aux = bool(want_aux)

    @staticmethod
    def args_from_train_config(train_config):
        """(scene, [sampling_net, shading_net], threshold, K) read from an initialised reference TrainConfig -- no device
        needed (tests/test_adapter_config.py runs this against the live reference).  A one-network run (plain NeRF,
        inFeatures = [RayMarchFromPoses]) gives [None, its net], and its depth_range is f_in[0]'s: without SpherePosDir the
        reference places and reports depth with the dataset's unwarped range (datasets.py:154-159)."""
        f1 = train_config.f_in[-1]
        info = train_config.dataset_info
        scene = dict(view_cell_center=list(info.view.view_cell_center), view_cell_size=list(info.view.view_cell_size),
                     depth_range=list(f1.depth_range), max_depth=float(f1.max_depth), fov=float(info.view.fov),
                     z_near=f1.z_near, z_far=f1.z_far)
        if getattr(f1, "useNDC", False):    # configs/*_ndc.ini: ndc_rays(self.h, self.w, self.view.focal, 1., ...) (features.py:430)
            scene.update(use_ndc=True, w=int(f1.w), h=int(f1.h), focal=float(info.view.focal))
        # posEnc / posEncArgs of each net, as its FeatureSet holds them (enc_type, n_freq_pos, n_freq_dir; features.py:326-339):
        # posEnc none ignores the band counts (-1 / -1).  The sampling net's fields take -1 for zero bands, since 0 there
        # means "the shading net's count".
        for f, (kp, kd), zero in ((f1, ("n_freq_pos", "n_freq_dir"), 0), (train_config.f_in[0], ("n_freq_pos0", "n_freq_dir0"), -1)):
            if hasattr(f, "enc_type"):
                p, d = (-1, -1) if f.enc_type == "none" else (int(f.n_freq_pos), int(f.n_freq_dir))
                scene.update({kp: p if p > 0 else min(p, zero), kd: d if d > 0 else min(d, zero)})
        thr = float(getattr(f1.z_sampler, "threshold", 0.0))   # FromClassifiedDepth and the linear samplers have none
        models = [train_config.models[0], train_config.models[1]] if len(train_config.models) > 1 else [None, train_config.models[0]]
        return scene, models, thr, int(f1.n_ray_samples)

    @staticmethod
    def sampler_from_train_config(train_config):
        """(sampler, pdf_transform) of the shading net's rayMarchSampler and losses[0] (src/nerf_raymarch_common.py:625-637):
        (1, 1 or 2) for FromClassifiedDepth, else (0, 1): the adaptive path.  Raises ValueError for a FromClassifiedDepth run
        whose losses[0] selects no transform.  A one-network run with LinearlySpacedZNearZFar (NoDepthRange) gives (2, 1)."""
        name = type(train_config.f_in[-1].z_sampler).__name__
        if len(train_config.f_in) == 1:
            if name not in LINEAR_SAMPLERS:
                raise ValueError(f"one-network runs need rayMarchSampler {' or '.join(LINEAR_SAMPLERS)}, not {name}")
            return 2, 1
        if name != "FromClassifiedDepth":
            return 0, 1
        loss0 = train_config.config_file.losses[0]
        if loss0 not in PDF_TRANSFORMS:
            raise ValueError(f"FromClassifiedDepth with losses[0] = {loss0} applies no transform to raw0 (not supported)")
        return 1, PDF_TRANSFORMS[loss0]

    @classmethod
    def from_train_config(cls, train_config, device=0):
        """Builds the renderer from an initialised reference TrainConfig (models, feature sets, dataset_info)."""
        scene, models, thr, k = cls.args_from_train_config(train_config)
        sampler, transform = cls.sampler_from_train_config(train_config)
        disc = getattr(train_config.f_in[-1].z_sampler, "disc", None)   # multiDepthFeatures[1] (nerf_raymarch_common.py:674-676)
        if models[0] is not None and disc is not None:
            sd = models[0].state_dict()
            last = max(int(n.split(".")[1]) for n in sd if n.startswith("layers.") and n.endswith(".weight"))
            width = int(sd[f"layers.{last}.weight"].shape[0])
            if width != int(disc):
                raise ValueError(f"the sampler places {disc} depth cells (multiDepthFeatures) but the sampling net has {width} outputs")
        return cls(scene, models[0], models[1], thr, k, device=device, sampler=sampler, pdf_transform=transform)

    def inference(self, batch_idx, gradient=False, **kwargs):
        if gradient:
            raise NotImplementedError("adanerf_b200 is an inference renderer (src/train.py is out of scope)")
        b = batch_idx.get_batch_input(1) if hasattr(batch_idx, "get_batch_input") else batch_idx
        pose, rot, dirs = b[KEY_POSE], b[KEY_ROT], b[KEY_DIRS]
        # [n_images, n_samples] batches (SpherePosDir.batch / RayMarchFromPoses.batch, features.py:392-427,845-864): one views
        # call, outputs view-major [n_images * n_samples, ...] like the reference's flattened ones
        kw = dict(want_nsamples=True, want_oracle_weights=self.want_oracle_weights,
                  want_aux=("weights", "alpha", "z_vals", "depth_est") if self.want_aux else False)
        if pose.shape[0] == 1:
            out = self.renderer.render_rays(pose[0], rot[0], dirs.reshape(-1, 3), self.threshold, self.K, **kw)
        else:
            out = self.renderer.render_views(pose.reshape(-1, 3), rot.reshape(-1, 3, 3), dirs.reshape(pose.shape[0], -1, 3),
                                             self.threshold, self.K, **kw)
        rgb = out["rgb"]
        if self.sampler == 2:   # one network: its dict only (TrainConfig.inference of a one-model run)
            d = {KEY_POST: rgb}
            if self.want_aux:
                d[KEY_WEIGHTS], d[KEY_ALPHA], d[KEY_ZVALS] = out["weights"], out["alpha"], out["z_vals"]
                d[KEY_DEPTH] = out["depth_est"].reshape(-1, 1)
            return [rgb], [d]
        raw0 = out["oracle_weights"]
        d0 = {KEY_POST: raw0, KEY_NET_OUT: raw0}
        d1 = {KEY_POST: rgb}
        if self.threshold > 0.0 and not self.sampler:
            d1[KEY_ASP] = out["n_samples"].to(torch.float32) / self.K
        if raw0 is not None and not self.sampler:
            d1[KEY_ORACLE] = raw0
        if self.want_aux:
            d1[KEY_WEIGHTS], d1[KEY_ALPHA], d1[KEY_ZVALS] = out["weights"], out["alpha"], out["z_vals"]
            d1[KEY_DEPTH] = out["depth_est"].reshape(-1, 1)   # features.py:576-577
        return [raw0, rgb], [d0, d1]

    __call__ = inference
