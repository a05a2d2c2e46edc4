"""ComfyUI graph nodes of the GGUF loader family, backed by the H100 kernels (importable only inside ComfyUI).

Drop-in contract (reference nodes.py:134-321): the six node keys, their widgets, RETURN_TYPES, FUNCTION names, the
"bootleg" category and the titles are unchanged, so saved workflows load as they are.  What the nodes hand to ComfyUI is this
package's `GGMLOps`, therefore every quantised Linear that comfy.sd instantiates runs `ggufb200_linear`.

The model patcher keeps the one behaviour the hot path relies on (reference nodes.py:43-47): a LoRA on a QUANTISED weight is
not baked into the packed bytes; the patch list is attached to the tensor (`tensor.patches`) and applied after the dequant on
every forward.  Dense (F16/F32) weights are patched the usual way.  `load()` forces `force_patch_weights=True` like the
reference (nodes.py:94-99): without it a partially loaded (lowvram) module would receive LowVramPatch objects in
`weight_function`, which the GGUF layers never read, and a LoRA on an offloaded quantised layer would be silently dropped.
Only the reference's mmap-release bounce (nodes.py:101-119) -- host memory policy -- is left out.
"""
import collections
import logging

import torch

import comfy.float
import comfy.lora
import comfy.model_management as mm
import comfy.model_patcher
import comfy.sd
import comfy.utils
import folder_paths
import nodes as comfy_nodes

from .dequant import is_quantized
from .loader import gguf_clip_loader, gguf_sd_loader
from .ops import GGMLOps, move_patch_to_device

DTYPE_WIDGET = ["default", "target", "float32", "float16", "bfloat16"]
_WeightBackup = collections.namedtuple("Dimension", ["weight", "inplace_update"])


def _register_gguf_folder(alias, fallbacks):
    """Expose `alias` as a file list restricted to *.gguf that shares the directories of the first known fallback key."""
    table = folder_paths.folder_names_and_paths
    previous = table.get(alias, ([], {}))[0]
    if not isinstance(previous, (list, set, tuple)):
        previous = []
    source = next((name for name in fallbacks if name in table), fallbacks[0])
    directories = table.get(source, ([], {}))[0]
    table[alias] = (directories or previous, {".gguf"})
    if previous and previous != directories:
        logging.warning(f"Unknown file list already present on key {alias}: {previous}")


_register_gguf_folder("unet_gguf", ["diffusion_models", "unet"])
_register_gguf_folder("clip_gguf", ["text_encoders", "clip"])


class GGUFModelPatcher(comfy.model_patcher.ModelPatcher):
    patch_on_device = False

    # -- quantised weights: keep the packed bytes, carry the patch list on the tensor
    def _attach_to_packed(self, key, weight, device_to):
        moved = weight.to(device_to)
        patch_home = self.load_device if self.patch_on_device else self.offload_device
        moved.patches = [(move_patch_to_device(self.patches[key], patch_home), key)]
        return moved

    # -- dense weights: fold the patches in, exactly like the stock patcher
    def _bake_into_dense(self, key, weight, device_to, inplace_update):
        if key not in self.backup:
            self.backup[key] = _WeightBackup(weight.to(device=self.offload_device, copy=inplace_update), inplace_update)
        if device_to is None:
            work = weight.to(torch.float32, copy=True)
        else:
            work = mm.cast_to_device(weight, device_to, torch.float32, copy=True)
        merged = comfy.lora.calculate_weight(self.patches[key], work, key)
        return comfy.float.stochastic_rounding(merged, weight.dtype)

    def patch_weight_to_device(self, key, device_to=None, inplace_update=False):
        if key not in self.patches:
            return
        weight = comfy.utils.get_attr(self.model, key)
        if is_quantized(weight):
            result = self._attach_to_packed(key, weight, device_to)
        else:
            inplace_update = self.weight_inplace_update or inplace_update
            result = self._bake_into_dense(key, weight, device_to, inplace_update)
        setter = comfy.utils.copy_to_param if inplace_update else comfy.utils.set_attr_param
        setter(self.model, key, result)

    def unpatch_model(self, device_to=None, unpatch_weights=True):
        if unpatch_weights:
            for param in self.model.parameters():
                if is_quantized(param) and getattr(param, "patches", None):
                    param.patches = []
        return super().unpatch_model(device_to=device_to, unpatch_weights=unpatch_weights)

    def load(self, *args, force_patch_weights=False, **kwargs):
        # quantised layers only understand `tensor.patches`: every patched key must go through patch_weight_to_device,
        # also for modules that stay on the offload device (reference nodes.py:94-99)
        return super().load(*args, force_patch_weights=True, **kwargs)

    def clone(self, *args, **kwargs):
        # The stock clone() copies ALL patcher state (wrappers, callbacks, hooks, attachments, pinned set ...) and builds the
        # twin with type(self); it is also called unbound on a plain ModelPatcher by the loader nodes (reference
        # nodes.py:121-132).  Borrow this class for the duration of the base-class clone instead of re-listing its fields.
        origin = self.__class__
        self.__class__ = GGUFModelPatcher
        try:
            twin = super().clone(*args, **kwargs)
        finally:
            self.__class__ = origin
        twin.__class__ = GGUFModelPatcher
        twin.patch_on_device = getattr(self, "patch_on_device", False)
        if origin is not GGUFModelPatcher:
            twin.size = 0          # sized by a foreign patcher class: recompute
        return twin


def _widget_to_dtype(choice):
    """'default'/None -> None (fp16 math), 'target' -> activation dtype, otherwise the named torch dtype."""
    if choice is None or choice == "default":
        return None
    return choice if choice == "target" else getattr(torch, choice)


def _gguf_unets():
    return list(folder_paths.get_filename_list("unet_gguf"))


class UnetLoaderGGUF:
    RETURN_TYPES = ("MODEL",)
    FUNCTION = "load_unet"
    CATEGORY = "bootleg"
    TITLE = "Unet Loader (GGUF)"

    @classmethod
    def INPUT_TYPES(cls):
        return {"required": {"unet_name": (_gguf_unets(),)}}

    def load_unet(self, unet_name, dequant_dtype=None, patch_dtype=None, patch_on_device=None):
        operations = GGMLOps()
        # deliberately CLASS attributes of GGMLOps.Linear, as in the reference (nodes.py:152-164)
        operations.Linear.dequant_dtype = _widget_to_dtype(dequant_dtype)
        operations.Linear.patch_dtype = _widget_to_dtype(patch_dtype)

        path = folder_paths.get_full_path("unet", unet_name)
        model = comfy.sd.load_diffusion_model_state_dict(gguf_sd_loader(path), model_options={"custom_operations": operations})
        if model is None:
            logging.error("ERROR UNSUPPORTED UNET {}".format(path))
            raise RuntimeError("ERROR: Could not detect model type of: {}".format(path))
        patcher = GGUFModelPatcher.clone(model)
        patcher.patch_on_device = patch_on_device
        return (patcher,)


class UnetLoaderGGUFAdvanced(UnetLoaderGGUF):
    TITLE = "Unet Loader (GGUF/Advanced)"

    @classmethod
    def INPUT_TYPES(cls):
        knobs = {name: (DTYPE_WIDGET, {"default": "default"}) for name in ("dequant_dtype", "patch_dtype")}
        return {"required": {"unet_name": (_gguf_unets(),), **knobs, "patch_on_device": ("BOOLEAN", {"default": False})}}


class CLIPLoaderGGUF:
    RETURN_TYPES = ("CLIP",)
    FUNCTION = "load_clip"
    CATEGORY = "bootleg"
    TITLE = "CLIPLoader (GGUF)"
    STOCK_NODE = "CLIPLoader"
    FILE_WIDGETS = ("clip_name",)

    @classmethod
    def get_filename_list(cls):
        return sorted(folder_paths.get_filename_list("clip") + folder_paths.get_filename_list("clip_gguf"))

    @classmethod
    def INPUT_TYPES(cls):
        required = {widget: (cls.get_filename_list(),) for widget in cls.FILE_WIDGETS}
        stock = getattr(comfy_nodes, cls.STOCK_NODE, None)
        stock_required = stock.INPUT_TYPES().get("required", {}) if stock is not None else {}
        if "type" in stock_required:
            required["type"] = stock_required["type"]
        return {"required": required}

    def load_data(self, ckpt_paths):
        state_dicts = []
        for path in ckpt_paths:
            if path.endswith(".gguf"):
                state_dicts.append(gguf_clip_loader(path))
                continue
            sd = comfy.utils.load_torch_file(path, safe_load=True)
            if "scaled_fp8" in sd:  # only one custom-ops family can be active per model
                raise NotImplementedError(
                    f"Mixing scaled FP8 with GGUF is not supported! Use regular CLIP loader or switch model(s)\n({path})")
            state_dicts.append(sd)
        return state_dicts

    def load_patcher(self, clip_paths, clip_type, clip_data):
        clip = comfy.sd.load_text_encoder_state_dicts(
            clip_type=clip_type,
            state_dicts=clip_data,
            model_options={"custom_operations": GGMLOps, "initial_device": mm.text_encoder_offload_device()},
            embedding_directory=folder_paths.get_folder_paths("embeddings"),
        )
        clip.patcher = GGUFModelPatcher.clone(clip.patcher)
        return clip

    def _load_files(self, names, type_name):
        paths = tuple(folder_paths.get_full_path("clip", name) for name in names)
        clip_type = getattr(comfy.sd.CLIPType, type_name.upper(), comfy.sd.CLIPType.STABLE_DIFFUSION)
        return (self.load_patcher(paths, clip_type, self.load_data(paths)),)

    def load_clip(self, clip_name, type="stable_diffusion"):
        return self._load_files((clip_name,), type)


class DualCLIPLoaderGGUF(CLIPLoaderGGUF):
    TITLE = "DualCLIPLoader (GGUF)"
    STOCK_NODE = "DualCLIPLoader"
    FILE_WIDGETS = ("clip_name1", "clip_name2")

    def load_clip(self, clip_name1, clip_name2, type):
        return self._load_files((clip_name1, clip_name2), type)


class TripleCLIPLoaderGGUF(CLIPLoaderGGUF):
    TITLE = "TripleCLIPLoader (GGUF)"
    STOCK_NODE = "TripleCLIPLoader"
    FILE_WIDGETS = ("clip_name1", "clip_name2", "clip_name3")

    def load_clip(self, clip_name1, clip_name2, clip_name3, type="sd3"):
        return self._load_files((clip_name1, clip_name2, clip_name3), type)


class QuadrupleCLIPLoaderGGUF(CLIPLoaderGGUF):
    TITLE = "QuadrupleCLIPLoader (GGUF)"
    STOCK_NODE = "QuadrupleCLIPLoader"
    FILE_WIDGETS = ("clip_name1", "clip_name2", "clip_name3", "clip_name4")

    def load_clip(self, clip_name1, clip_name2, clip_name3, clip_name4, type="stable_diffusion"):
        return self._load_files((clip_name1, clip_name2, clip_name3, clip_name4), type)


NODE_CLASS_MAPPINGS = {
    cls.__name__: cls
    for cls in (UnetLoaderGGUF, CLIPLoaderGGUF, DualCLIPLoaderGGUF, TripleCLIPLoaderGGUF, QuadrupleCLIPLoaderGGUF, UnetLoaderGGUFAdvanced)
}
