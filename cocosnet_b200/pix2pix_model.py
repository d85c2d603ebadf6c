"""Pix2PixModel with the reference's public surface (models/pix2pix_model.py):
forward(data, mode, GforD=None, alpha=1), create_optimizers, save, and
.net ModuleDict {netG, netD, netCorr, netDomainClassifier}.  One process per
GPU: the model lives on the current CUDA device."""
import os

import torch
import torch.nn.functional as F

from . import nets as networks
from . import util


class Pix2PixModel(torch.nn.Module):
    @staticmethod
    def modify_commandline_options(parser, is_train):
        networks.modify_commandline_options(parser, is_train)
        return parser

    def __init__(self, opt):
        super().__init__()
        self.opt = opt
        self.alpha = 1
        self.after_netG_backward = None  # trainer hook: called once the backward has left netG (its gradients are final)
        self.free_inference_graph()
        self.infer_graph_error = None
        self.net = torch.nn.ModuleDict(self.initialize_networks(opt))
        if opt.isTrain:
            self.vggnet_fix = networks.VGG19_feature_color_torchversion(vgg_normal_correct=opt.vgg_normal_correct)
            vgg_path = getattr(opt, "vgg_path", "models/vgg19_conv.pth")
            if os.path.exists(vgg_path):
                self.vggnet_fix.load_state_dict(torch.load(vgg_path, map_location="cpu"))
            elif not getattr(opt, "allow_random_vgg", False):
                raise FileNotFoundError(
                    "%s not found (reference pix2pix_model.py:30 loads it); pass opt.allow_random_vgg=True for "
                    "synthetic benchmarking with a seeded random VGG" % vgg_path)
            self.vggnet_fix.eval()
            for p in self.vggnet_fix.parameters():
                p.requires_grad = False
            if self.use_gpu():
                self.vggnet_fix.cuda()
            self.contextual_forward_loss = networks.ContextualLoss_forward(opt)
            self.criterionGAN = networks.GANLoss(opt.gan_mode, opt=opt)
            self.criterionFeat = torch.nn.L1Loss()
            self.MSE_loss = torch.nn.MSELoss()
            self.perceptual_layer = {"5_2": -1, "4_2": -2}[opt.which_perceptual]

    # ------------------------------------------------------------------ API
    def forward(self, data, mode, GforD=None, alpha=1):
        input_label, input_semantics, real_image, self_ref, ref_image, ref_label, ref_semantics = \
            self.preprocess_input(data)
        self.alpha = alpha
        if mode == "generator":
            g_loss, gen = self.compute_generator_loss(input_label, input_semantics, real_image, ref_label,
                                                      ref_semantics, ref_image, self_ref)
            out = {"fake_image": gen["fake_image"], "input_semantics": input_semantics,
                   "ref_semantics": ref_semantics}
            for k in ("warp_out", "warp_mask", "adaptive_feature_seg", "adaptive_feature_img", "warp_cycle",
                      "warp_i2r", "warp_i2r2i"):
                out[k] = gen.get(k)
            return g_loss, out
        if mode == "discriminator":
            return self.compute_discriminator_loss(input_semantics, real_image, GforD, label=input_label)
        if mode == "inference":
            with torch.no_grad():
                out = self.inference(input_semantics, ref_semantics=ref_semantics, ref_image=ref_image,
                                     self_ref=self_ref)
            out["input_semantics"] = input_semantics
            out["ref_semantics"] = ref_semantics
            return out
        raise ValueError("|mode| is invalid")

    # ------------------------------------------------------------------ CUDA-graph inference
    def run_inference(self, data):
        """`self(data, mode="inference")`, replayed from one CUDA graph: the same keys and the same bits.  On a CUDA
        model in eval() the first call for an input signature (the batch's shapes plus the identity and address of
        every parameter and buffer of netG and netCorr) runs eagerly as warm-up, the next call with that signature
        captures the forward, and from then on a call copies the batch into static device buffers and replays the
        graph: one launch in place of the forward's per-op dispatch.  One signature is kept: a batch of other shapes
        (test.py's short last batch) runs eagerly.  Weights updated in place (load_state_dict, an optimiser step) are
        read by the replay; replacing a parameter tensor re-captures.
        Eager always on the CPU, in train(), under COCOS_CUDA_GRAPH=0, and with --noise_for_mask / --mask_noise,
        whose random draws a replay would not repeat.  The returned tensors are copies: a later call does not
        overwrite them."""
        self.check_glasses_slot(data)  # the capture skips preprocess_input's host-side assertion: check it here
        if not self.inference_graph_capable():
            return self(data, mode="inference")
        shapes = tuple((k, tuple(v.shape), v.dtype) for k, v in sorted(data.items()) if torch.is_tensor(v))
        key = (shapes, self._weights_key())
        if self._infer["graph"] is not None and key != self._infer["key"]:
            if shapes != self._infer["key"][0]:
                return self(data, mode="inference")  # not the captured shapes
            self.free_inference_graph()  # a parameter or buffer was replaced: warm up and capture again
        if self._infer["graph"] is None:
            if key != self._infer["warm_key"]:
                self._infer["warm_key"] = key
                return self(data, mode="inference")
            self._capture_inference(data, key)
            if self._infer["graph"] is None:  # capture failed: stay eager, loudly
                return self(data, mode="inference")
        g = self._infer
        for k, buf in g["static_in"].items():
            buf.copy_(data[k], non_blocking=True)
        g["graph"].replay()
        return {k: (v.clone() if torch.is_tensor(v) else v) for k, v in g["static_out"].items()}

    def inference_graph_capable(self):
        opt = self.opt
        return (not self.training and next(self.net["netG"].parameters()).is_cuda and self.use_gpu()
                and os.environ.get("COCOS_CUDA_GRAPH", "1") == "1" and self.infer_graph_error is None
                and not getattr(opt, "noise_for_mask", False) and not getattr(opt, "mask_noise", False))

    def free_inference_graph(self):
        """Drop the captured inference forward and its private memory pool."""
        self._infer = {"graph": None, "key": None, "warm_key": None, "static_in": None, "static_out": None}

    def _weights_key(self):
        nets = (self.net["netG"], self.net["netCorr"])
        return tuple((id(t), t.data_ptr()) for n in nets for t in list(n.parameters()) + list(n.buffers()))

    def _capture_inference(self, data, key):
        from . import nhwc
        static_in = {k: torch.empty_like(v, device="cuda") for k, v in data.items() if torch.is_tensor(v)}
        for k, buf in static_in.items():
            buf.copy_(data[k], non_blocking=True)
        static = dict(data)
        static.update(static_in)
        torch.cuda.synchronize()
        graph = torch.cuda.CUDAGraph()
        # everything the graph reads must be produced inside it (or be immutable): the weight packs are re-made by
        # every replay from the parameters' storage, which is what makes in-place weight updates visible to it
        nhwc.clear_pack_cache()
        try:
            with torch.no_grad(), torch.cuda.graph(graph):  # captured on torch.cuda.graph's side stream
                out = self(static, mode="inference")
        except Exception as e:  # noqa: BLE001 -- an op that cannot be captured: report it and keep running eagerly
            self.infer_graph_error = "%s: %s" % (type(e).__name__, str(e).splitlines()[0] if str(e) else "")
            print("cocosnet_b200: CUDA-graph capture of inference failed (%s); running eagerly" % self.infer_graph_error)
            if os.environ.get("COCOS_GRAPH_TRACE", "0") == "1":
                import traceback
                traceback.print_exc()
            torch.cuda.synchronize()
            nhwc.clear_pack_cache()
            return
        nhwc.clear_pack_cache()  # buffers packed during the capture live in the graph's pool: not for eager use
        self._infer = {"graph": graph, "key": key, "warm_key": None, "static_in": static_in, "static_out": out}

    def check_glasses_slot(self, data):
        """celebahq: preprocess_input's assertion that no pixel has the id of the glasses slot (semantic_nc - 3, which
        the glasses channel fills), on the host batch -- a captured forward cannot run it, so run_inference does it on
        every path before the batch reaches the GPU.  Raises the same AssertionError."""
        if self.opt.dataset_mode != "celebahq":
            return
        slot = self.opt.semantic_nc - 3
        assert not bool((data["label"][:, ::2].long() == slot).any())
        assert not bool((data["label_ref"][:, ::2].long() == slot).any())

    def create_optimizers(self, opt):
        G_params = [{"params": self.net["netG"].parameters(), "lr": opt.lr * 0.5},
                    {"params": self.net["netCorr"].parameters(), "lr": opt.lr * 0.5}]
        D_params = []
        if opt.isTrain:
            D_params += list(self.net["netD"].parameters())
            if opt.weight_domainC > 0 and opt.domain_rela:
                D_params += list(self.net["netDomainClassifier"].parameters())
        if opt.no_TTUR:
            beta1, beta2, G_lr, D_lr = opt.beta1, opt.beta2, opt.lr, opt.lr
        else:
            beta1, beta2, G_lr, D_lr = 0.0, 0.9, opt.lr / 2, opt.lr * 2
        fused = self.use_gpu()
        opt_G = torch.optim.Adam(G_params, lr=G_lr, betas=(beta1, beta2), eps=1e-3, fused=fused)
        opt_D = torch.optim.Adam(D_params, lr=D_lr, betas=(beta1, beta2), fused=fused)
        return opt_G, opt_D

    def save(self, epoch):
        util.save_network(self.net["netG"], "G", epoch, self.opt)
        util.save_network(self.net["netD"], "D", epoch, self.opt)
        util.save_network(self.net["netCorr"], "Corr", epoch, self.opt)
        if self.opt.weight_domainC > 0 and self.opt.domain_rela:
            util.save_network(self.net["netDomainClassifier"], "DomainClassifier", epoch, self.opt)

    # -------------------------------------------------------------- helpers
    def initialize_networks(self, opt):
        net = {"netG": networks.define_G(opt), "netD": networks.define_D(opt) if opt.isTrain else None,
               "netCorr": networks.define_Corr(opt),
               "netDomainClassifier": networks.define_DomainClassifier(opt)
               if opt.weight_domainC > 0 and opt.domain_rela else None}
        if not opt.isTrain or opt.continue_train:
            net["netG"] = util.load_network(net["netG"], "G", opt.which_epoch, opt)
            if opt.isTrain:
                net["netD"] = util.load_network(net["netD"], "D", opt.which_epoch, opt)
            net["netCorr"] = util.load_network(net["netCorr"], "Corr", opt.which_epoch, opt)
            if opt.weight_domainC > 0 and opt.domain_rela:
                net["netDomainClassifier"] = util.load_network(net["netDomainClassifier"], "DomainClassifier",
                                                               opt.which_epoch, opt)
            if (not opt.isTrain) and opt.use_ema:
                net["netG"] = util.load_network(net["netG"], "G_ema", opt.which_epoch, opt)
                net["netCorr"] = util.load_network(net["netCorr"], "netCorr_ema", opt.which_epoch, opt)
        return net

    def use_gpu(self):
        return len(self.opt.gpu_ids) > 0

    def _dev(self, t):
        return t.cuda(non_blocking=True) if self.use_gpu() else t

    def preprocess_input(self, data):
        """pix2pix_model.py:144-194: device move + one-hot label maps."""
        mode = self.opt.dataset_mode
        data = dict(data)
        glasses = glasses_ref = input_semantics = ref_semantics = None
        if mode == "celebahq":
            glasses = self._dev(data["label"][:, 1::2]).long()
            data["label"] = data["label"][:, ::2]
            glasses_ref = self._dev(data["label_ref"][:, 1::2]).long()
            data["label_ref"] = data["label_ref"][:, ::2]
        elif mode in ("celebahqedge", "deepfashion"):
            keep = 1 if mode == "celebahqedge" else 3
            input_semantics = self._dev(data["label"]).clone().float()
            data["label"] = data["label"][:, :keep]
            ref_semantics = self._dev(data["label_ref"]).clone().float()
            data["label_ref"] = data["label_ref"][:, :keep]
        for k in ("label", "image", "ref", "label_ref", "self_ref"):
            data[k] = self._dev(data[k])
        if mode != "deepfashion":
            data["label"] = data["label"].long()
            data["label_ref"] = data["label_ref"].long()
        if mode not in ("celebahqedge", "deepfashion"):
            nc = self.opt.label_nc + (1 if self.opt.contain_dontcare_label else 0)
            bs, _, h, w = data["label"].shape
            zeros = lambda: torch.zeros(bs, nc, h, w, dtype=torch.float32, device=data["label"].device)  # noqa: E731
            input_semantics = zeros().scatter_(1, data["label"], 1.0)
            ref_semantics = zeros().scatter_(1, data["label_ref"], 1.0)
        if mode == "celebahq":
            # pix2pix_model.py:186-190 asserts that the glasses slot is empty; a host read cannot be captured into a
            # CUDA graph, so the check only runs outside a capture (the eager warm-up iterations see the same data)
            if not (input_semantics.is_cuda and torch.cuda.is_current_stream_capturing()):
                assert input_semantics[:, -3:-2].sum().item() == 0
                assert ref_semantics[:, -3:-2].sum().item() == 0
            input_semantics[:, -3:-2] = glasses
            ref_semantics[:, -3:-2] = glasses_ref
        if getattr(self.opt, "channels_last", False) and self.use_gpu():
            cl = torch.channels_last
            input_semantics = input_semantics.contiguous(memory_format=cl)
            ref_semantics = ref_semantics.contiguous(memory_format=cl)
            data["image"] = data["image"].contiguous(memory_format=cl)
            data["ref"] = data["ref"].contiguous(memory_format=cl)
        return (data["label"], input_semantics, data["image"], data["self_ref"], data["ref"], data["label_ref"],
                ref_semantics)

    def get_ctx_loss(self, source, target):  # pix2pix_model.py:196-203
        ctx = self.contextual_forward_loss
        total = torch.mean(ctx(source[-1], target[-1].detach())) * 8
        total = total + torch.mean(ctx(source[-2], target[-2].detach())) * 4
        total = total + torch.mean(ctx(F.avg_pool2d(source[-3], 2), F.avg_pool2d(target[-3].detach(), 2))) * 2
        if self.opt.use_22ctx:
            total = total + torch.mean(ctx(F.avg_pool2d(source[-4], 4), F.avg_pool2d(target[-4].detach(), 4)))
        return total

    def _sample_weights(self, self_ref):  # pix2pix_model.py:227,249 (per-replica normalisation)
        s = self_ref[:, 0, 0, 0]
        return (s / (s.sum() + 1e-5)).view(-1, 1, 1, 1)

    def compute_generator_loss(self, input_label, input_semantics, real_image, ref_label=None, ref_semantics=None,
                               ref_image=None, self_ref=None):
        opt = self.opt
        G_losses = {}
        gen = self.generate_fake(input_semantics, real_image, ref_semantics=ref_semantics, ref_image=ref_image,
                                 self_ref=self_ref)
        if gen.get("loss_novgg_featpair") is not None:
            G_losses["no_vgg_feat"] = gen["loss_novgg_featpair"]
        if opt.warp_cycle_w > 0:
            ref = ref_image if opt.warp_patch else F.avg_pool2d(ref_image, opt.warp_stride)
            G_losses["G_warp_cycle"] = F.l1_loss(gen["warp_cycle"], ref) * opt.warp_cycle_w
            if opt.two_cycle:
                real = F.avg_pool2d(real_image, opt.warp_stride)
                G_losses["G_warp_cycle"] = G_losses["G_warp_cycle"] + \
                    F.l1_loss(gen["warp_i2r2i"], real) * opt.warp_cycle_w
        if opt.warp_self_w > 0:
            sw = self._sample_weights(self_ref)
            G_losses["G_warp_self"] = torch.mean(F.l1_loss(gen["warp_out"], real_image, reduction="none") * sw) \
                * opt.warp_self_w

        pred_fake, pred_real, extra, _, _ = self.discriminate(input_semantics, gen["fake_image"], real_image)
        G_losses["GAN"] = self.criterionGAN(pred_fake, True, for_discriminator=False) * opt.weight_gan
        if not opt.no_ganFeat_loss and isinstance(extra, dict) and extra.get("GAN_Feat") is not None:
            G_losses["GAN_Feat"] = extra["GAN_Feat"]
        elif not opt.no_ganFeat_loss:
            num_D = len(pred_fake)
            feat = torch.zeros(1, device=real_image.device)
            for i in range(num_D):
                for j in range(len(pred_fake[i]) - 1):  # last output is the prediction itself
                    feat = feat + self.criterionFeat(pred_fake[i][j], pred_real[i][j].detach()) * opt.lambda_feat / num_D
            G_losses["GAN_Feat"] = feat

        keys = ["r12", "r22", "r32", "r42", "r52"]
        sw = self._sample_weights(self_ref)
        fm_w = dict(zip(keys, [1.0 / 32, 1.0 / 16, 1.0 / 8, 1.0 / 4, 1.0]))
        if gen.get("real_features_nt") is not None:
            # one recorded VGG19 pass: the feature (weighted L1) and perceptual (MSE) losses are accumulated on the fp16
            # NHWC features against the real image's, only what the contextual loss reads is unpacked
            from .nets import fast as _fast
            from .nets.correspondence import _VGG_CFG
            from .util import vgg_preprocess
            ctx_keys = keys[-4:] if opt.use_22ctx else keys[-3:]
            x = vgg_preprocess(gen["fake_image"], vgg_normal_correct=self.vggnet_fix.vgg_normal_correct)
            ctx_feats, l1, mse = _fast.vgg_forward_losses(
                self.vggnet_fix, x, _VGG_CFG, gen["real_features_nt"],
                {k: w * opt.lambda_vgg * opt.fm_ratio for k, w in fm_w.items()}, sw,
                {keys[self.perceptual_layer]: opt.weight_perceptual}, ctx_keys)
            G_losses["fm"], G_losses["perc"] = l1.reshape(()), mse.reshape(())
            fake_features = [None] * (len(keys) - len(ctx_keys)) + list(ctx_feats)
        else:
            fake_features = self.vggnet_fix(gen["fake_image"], keys, preprocess=True)
            loss = 0
            for k, ff, rf in zip(keys, fake_features, gen["real_features"]):
                loss = loss + fm_w[k] * util.weighted_l1_loss(ff, rf.detach(), sw)
            G_losses["fm"] = loss * opt.lambda_vgg * opt.fm_ratio
            G_losses["perc"] = util.mse_loss(fake_features[self.perceptual_layer],
                                             gen["real_features"][self.perceptual_layer].detach()) * opt.weight_perceptual
        G_losses["contextual"] = self.get_ctx_loss(fake_features, gen["ref_features"]) * opt.lambda_vgg * opt.ctx_w

        if opt.warp_mask_losstype != "none":  # pix2pix_model.py:261-276
            ref_l = F.interpolate(ref_label.float(), scale_factor=0.25, mode="nearest").long().squeeze(1)
            gt_l = F.interpolate(input_label.float(), scale_factor=0.25, mode="nearest").long().squeeze(1)
            nc = gen["warp_mask"].shape[1]
            # weight 0 for gt classes absent from the exemplar and for class 0 -- same rule, no host sync
            present = torch.zeros(ref_l.shape[0], nc, device=ref_l.device).scatter_(1, ref_l.flatten(1), 1.0)
            weights = present.gather(1, gt_l.flatten(1)).view_as(gt_l).float()
            weights = weights * (gt_l != 0).float()
            nll = F.nll_loss(torch.log(gen["warp_mask"] + 1e-10), gt_l, reduction="none")
            G_losses["mask"] = (nll * weights).sum() / (weights.sum() + 1e-5) * opt.weight_mask
        return G_losses, gen

    def compute_discriminator_loss(self, input_semantics, real_image, GforD, label=None):
        # the reference marks the detached fake as requiring grad (pix2pix_model.py:285-286) although nothing
        # reads that gradient; leaving it off skips a useless input-gradient pass through D.
        fake_image = GforD["fake_image"].detach()
        # the hinge loss only reads the final predictions: no feature outputs in the D step
        pred_fake, pred_real, _, _, _ = self.discriminate(input_semantics, fake_image, real_image, need_feats=False)
        return {"D_Fake": self.criterionGAN(pred_fake, False, for_discriminator=True) * self.opt.weight_gan,
                "D_real": self.criterionGAN(pred_real, True, for_discriminator=True) * self.opt.weight_gan}

    def _cbn_in(self, coor_out, input_semantics):
        kind = self.opt.CBN_intype
        if kind == "mask":
            return input_semantics
        if kind == "warp":
            return coor_out["warp_out"]
        return torch.cat((coor_out["warp_out"], input_semantics), dim=1)

    def generate_fake(self, input_semantics, real_image, ref_semantics=None, ref_image=None, self_ref=None):
        keys = ["r12", "r22", "r32", "r42", "r52"]
        # only the layers the contextual loss reads (pix2pix_model.py:196-203 indexes them from the end)
        ctx_keys = keys[-4:] if self.opt.use_22ctx else keys[-3:]
        gen = {"ref_features": self.vggnet_fix(ref_image, ctx_keys, preprocess=True)}
        coor_out = self.net["netCorr"](ref_image, real_image, input_semantics, ref_semantics, alpha=self.alpha)
        if self.after_netG_backward is not None and coor_out["warp_out"].requires_grad:
            # the gradient of netCorr's output is complete only after netG's whole backward (netG reads warp_out);
            # autograd runs the parameters' AccumulateGrad nodes before it continues upstream
            fire = self.after_netG_backward

            def _hook(g):
                fire()
                return g
            coor_out["warp_out"].register_hook(_hook)
        from .nets import fast as _fast
        if _fast.fused_losses() and _fast.vgg_supported(self.vggnet_fix, real_image):
            # the real image's VGG features stay fp16 NHWC: targets of the fused feature / perceptual losses
            from .nets.correspondence import _VGG_CFG
            from .util import vgg_preprocess
            gen["real_features_nt"] = _fast.vgg_features_nt(
                self.vggnet_fix, vgg_preprocess(real_image, vgg_normal_correct=self.vggnet_fix.vgg_normal_correct), keys,
                _VGG_CFG)
        else:
            gen["real_features"] = self.vggnet_fix(real_image, keys, preprocess=True)
        gen["fake_image"] = self.net["netG"](input_semantics, warp_out=self._cbn_in(coor_out, input_semantics))
        return {**gen, **coor_out}

    def inference(self, input_semantics, ref_semantics=None, ref_image=None, self_ref=None):
        coor_out = self.net["netCorr"](ref_image, None, input_semantics, ref_semantics, alpha=self.alpha)
        gen = {"fake_image": self.net["netG"](input_semantics, warp_out=self._cbn_in(coor_out, input_semantics))}
        return {**gen, **coor_out}

    def discriminate(self, input_semantics, fake_image, real_image, need_feats=True):
        from .nets import fast as _fast
        if _fast.discriminator_supported(self.net["netD"], input_semantics, real_image):
            # [semantics | image] pairs packed straight into the fp16 NHWC input of the PatchGANs (no fp32 concat)
            pred_fake, pred_real, feat_loss = _fast.discriminator_forward(self.net["netD"], input_semantics, fake_image,
                                                                          real_image, need_feats=need_feats)
            # feat_loss: the feature-matching loss already accumulated on the NHWC features (generator step)
            return pred_fake, pred_real, {"GAN_Feat": feat_loss}, None, None
        fake_and_real = torch.cat([torch.cat([input_semantics, fake_image], dim=1),
                                   torch.cat([input_semantics, real_image], dim=1)], dim=0)
        d_out, seg, cam_logit = self.net["netD"](fake_and_real)
        pred_fake, pred_real = self.divide_pred(d_out)
        fake_cam = real_cam = None
        if self.opt.D_cam > 0:
            fake_cam = torch.cat([it[:it.shape[0] // 2] for it in cam_logit], dim=1)
            real_cam = torch.cat([it[it.shape[0] // 2:] for it in cam_logit], dim=1)
        return pred_fake, pred_real, seg, fake_cam, real_cam

    @staticmethod
    def divide_pred(pred):
        if isinstance(pred, list):
            fake = [[t[:t.size(0) // 2] for t in p] for p in pred]
            real = [[t[t.size(0) // 2:] for t in p] for p in pred]
            return fake, real
        return pred[:pred.size(0) // 2], pred[pred.size(0) // 2:]
