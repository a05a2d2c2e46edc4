"""ggufb200: H100-native (sm_90a) drop-in for the dequant + Linear hot path of city96/ComfyUI-GGUF.

ComfyUI imports this directory as a custom node package and reads NODE_CLASS_MAPPINGS / NODE_DISPLAY_NAME_MAPPINGS from it.
Outside ComfyUI (tests, benchmarks, the GPU box) the host packages are absent and only the kernel-facing modules
(`dequant`, `ops`, `loader`, `replicas`) are used, through `__graft_entry__.load_package()`.
"""
import importlib.util as _ilu


def _inside_comfyui() -> bool:
    return all(_ilu.find_spec(name) is not None for name in ("comfy", "folder_paths", "nodes"))


if _inside_comfyui():  # pragma: no cover - needs a ComfyUI checkout
    from . import nodes as _nodes

    NODE_CLASS_MAPPINGS = dict(_nodes.NODE_CLASS_MAPPINGS)
    NODE_DISPLAY_NAME_MAPPINGS = {key: cls.TITLE for key, cls in NODE_CLASS_MAPPINGS.items()}
    __all__ = ["NODE_CLASS_MAPPINGS", "NODE_DISPLAY_NAME_MAPPINGS"]
