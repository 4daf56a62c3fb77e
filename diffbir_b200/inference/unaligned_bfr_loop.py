"""UnAlignedBFRInferenceLoop (reference: diffbir/inference/unaligned_bfr_loop.py): restoration of whole photos that
contain faces. Every face is detected (RetinaFace), aligned to the 512 FFHQ template and restored with the face
SwinIR pipeline; the photo itself goes through the background pipeline (v2: BSRNet, v2.1: SwinIR on the bicubic
up-scaled input); then each sample's restored faces are pasted back through their ParseNet masks.

Output layout under --output: restored_faces/{stem}_face_{i}_{k}.png, cropped_faces/ (under the last restored-face
name of that face, as the reference writes it), restored_backgrounds/{stem}_{k}.png, {stem}_{k}.png and prompt.csv.
An image without a detected face writes only its prompt.csv row, as in the reference."""
from typing import Generator, List

import numpy as np
import torch
from PIL import Image

from ..pipeline import BSRNetPipeline, SwinIRPipeline
from ..utils.common import instantiate_from_config
from ..utils.face import FaceRestoreHelper
from .loop import InferenceLoop, load_checkpoint, load_config
from .pretrained_models import resolve


class UnAlignedBFRInferenceLoop(InferenceLoop):
    def load_cleaner(self) -> None:
        from .. import arch
        from ..utils import synth
        v = self.args.version
        if v == "v1":
            raise ValueError("DiffBIR v1 doesn't support unaligned BFR, please use v2 or v2.1.")
        if v == "v2":
            yaml_name, shapes, key = "bsrnet.yaml", arch.rrdbnet_shapes(arch.RRDBNET_CFG), "bsrnet"
        else:
            yaml_name, shapes, key = "swinir.yaml", arch.swinir_shapes(arch.SWINIR_CFG), "swinir_realesrgan"
        self.bg_cleaner = instantiate_from_config(load_config(yaml_name), device=self.args.device)
        self.face_cleaner = instantiate_from_config(load_config("swinir.yaml"), device=self.args.device)
        if self.synthetic:
            self.bg_cleaner.load_state_dict(synth.make_state_dict(shapes, self.args.seed + 4))
            self.face_cleaner.load_state_dict(synth.make_state_dict(arch.swinir_shapes(arch.SWINIR_CFG),
                                                                    self.args.seed + 5))
        else:
            self.bg_cleaner.load_state_dict(load_checkpoint(resolve(key, self.weights_dir)), strict=True)
            self.face_cleaner.load_state_dict(load_checkpoint(resolve("swinir_face", self.weights_dir)), strict=True)

    def load_pipeline(self) -> None:
        a = self.args
        if a.version == "v2":
            bg = BSRNetPipeline(self.bg_cleaner, self.cldm, self.diffusion, self.cond_fn, a.device, a.upscale)
            self.bg_requires_upscale = False
        else:
            bg = SwinIRPipeline(self.bg_cleaner, self.cldm, self.diffusion, self.cond_fn, a.device)
            self.bg_requires_upscale = True
        self.pipeline_dict = {"background": bg,
                              "face": SwinIRPipeline(self.face_cleaner, self.cldm, self.diffusion, self.cond_fn, a.device)}

    def pipelines(self) -> list:
        return list(self.pipeline_dict.values())

    def face_networks(self):
        """(detector, parser) callables of FaceRestoreHelper, on the engines. The parser returns device tensors, so the
        paste-back runs on the engine too."""
        from .. import arch
        from ..engine.parsenet import ParseNetEngine
        from ..engine.retinaface import RetinaFaceEngine
        if self.synthetic:
            from ..utils.synth import synthetic_face_nets
            det_sd, parse_sd = synthetic_face_nets(self.args.seed)
        else:
            det_sd = arch.retinaface_state_dict(load_checkpoint(resolve("retinaface_resnet50", self.weights_dir)))
            parse_sd = arch.parsenet_state_dict(load_checkpoint(resolve("parsenet", self.weights_dir)))
        det = RetinaFaceEngine(det_sd, device=self.args.device)
        parse = ParseNetEngine(parse_sd, device=self.args.device)
        return det.candidates, parse.masks_device

    def setup(self) -> None:
        import os
        super().setup()
        self.cropped_face_dir = os.path.join(self.save_dir, "cropped_faces")
        self.restored_face_dir = os.path.join(self.save_dir, "restored_faces")
        self.restored_bg_dir = os.path.join(self.save_dir, "restored_backgrounds")
        for d in (self.cropped_face_dir, self.restored_face_dir, self.restored_bg_dir):
            os.makedirs(d, exist_ok=True)
        detector, parser = self.face_networks()
        self.face_helper = FaceRestoreHelper(self.args.device, upscale_factor=1, face_size=512, use_parse=True,
                                             det_model="retinaface_resnet50", detector=detector, parser=parser)
        self.face_samples: List[List[np.ndarray]] = []

    def load_lq(self) -> Generator[Image.Image, None, None]:
        for lq in super().load_lq():
            self.face_helper.clean_all()
            self.face_samples.clear()
            upscaled_bg = np.array(lq.resize(tuple(int(x * self.args.upscale) for x in lq.size), Image.BICUBIC))
            self.face_helper.read_image(upscaled_bg)        # RGB, used as the detector's BGR (as in the reference)
            self.face_helper.get_face_landmarks_5(resize=640, eye_dist_threshold=5)
            self.face_helper.align_warp_face()
            print(f"detect {len(self.face_helper.cropped_faces)} faces")
            for i, lq_face in enumerate(self.face_helper.cropped_faces):
                self.loop_ctx["is_face"] = True
                self.loop_ctx["face_idx"] = i
                self.loop_ctx["cropped_face"] = lq_face
                yield Image.fromarray(lq_face)
            self.loop_ctx["is_face"] = False
            yield lq

    def after_load_lq(self, lq: Image.Image) -> np.ndarray:
        if self.loop_ctx["is_face"]:
            self.pipeline = self.pipeline_dict["face"]
        else:
            self.pipeline = self.pipeline_dict["background"]
            if self.bg_requires_upscale:
                lq = lq.resize(tuple(int(x * self.args.upscale) for x in lq.size), Image.BICUBIC)
        return super().after_load_lq(lq)

    def save(self, samples: List[np.ndarray], pos_prompt: str, neg_prompt: str) -> None:
        import os
        stem = self.loop_ctx["file_stem"]
        is_face = self.loop_ctx["is_face"]
        self.prompt_row(f"{stem}_face_{self.loop_ctx['face_idx']}" if is_face else stem, pos_prompt, neg_prompt)
        if is_face:
            face_idx = self.loop_ctx["face_idx"]
            for i, sample in enumerate(samples):
                file_name = f"{stem}_face_{face_idx}_{i}.png"
                Image.fromarray(sample).save(os.path.join(self.restored_face_dir, file_name))
            # the reference saves the cropped face under the last restored-face name of this face
            Image.fromarray(self.loop_ctx["cropped_face"]).save(os.path.join(self.cropped_face_dir, file_name))
            self.face_samples.append(samples)
            return
        helper = self.face_helper
        helper.get_inverse_affine()
        per_sample = list(map(list, zip(*self.face_samples)))          # [sample k][face i]
        masks = helper.parse_faces([f for faces in per_sample for f in faces])    # one batched parse
        n_faces = len(self.face_samples)
        if isinstance(masks, torch.Tensor):        # engine masks: every sample pasted on the device in one call
            for k, (restored, restored_bg) in enumerate(zip(helper.paste_faces_device(samples, per_sample, masks),
                                                            samples)):
                file_name = f"{stem}_{k}.png"
                Image.fromarray(restored_bg).save(os.path.join(self.restored_bg_dir, file_name))
                Image.fromarray(restored).save(os.path.join(self.save_dir, file_name))
            return
        for k, (faces, restored_bg) in enumerate(zip(per_sample, samples)):
            for face in faces:
                helper.add_restored_face(face)
            restored = helper.paste_faces_to_input_image(restored_bg, masks[k * n_faces:(k + 1) * n_faces])
            file_name = f"{stem}_{k}.png"
            Image.fromarray(restored_bg).save(os.path.join(self.restored_bg_dir, file_name))
            Image.fromarray(restored).save(os.path.join(self.save_dir, file_name))
            helper.restored_faces.clear()
