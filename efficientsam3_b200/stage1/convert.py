"""Checkpoint key contracts between stage 1 and the assembled EfficientSAM3 model (SURVEY.md section 8f, row N4) -- pure
dictionary work, no tensors are touched:

  merge_student_into_sam3   stage1/convert_image_encoder_weights_stage1.py:12-21, 96-141: a stage-1 student state_dict is normalised
                            (`module.`, `student_trunk.`, already-merged prefixes stripped), re-rooted under
                            `detector.backbone.vision_backbone.trunk.model.` and laid over a full SAM3 checkpoint whose own trunk
                            weights are dropped
  merge_text_student_into_sam3
                            stage1/convert_text_encoder_weights_stage1.py:8-19, 102-163: the same for a stage-1 text student
                            (`module.`, `detector.backbone.language_backbone.`, `backbone.language_backbone.` stripped), re-rooted
                            under `detector.backbone.language_backbone.`; the teacher's keys under the replace prefix are dropped
  clean_merged_keys         sam3/sam3/model_builder.py:594-612 (`_load_checkpoint`): `detector.` and `student_trunk.` removed, so the
                            result loads into efficientsam3_b200.model_builder modules (`backbone.vision_backbone.trunk.model.*`)
"""
from __future__ import annotations

_STUDENT_PREFIXES = ("module.", "student_trunk.", "detector.backbone.vision_backbone.trunk.model.",
                     "detector.backbone.vision_backbone.trunk.", "backbone.vision_backbone.trunk.model.",
                     "backbone.vision_backbone.trunk.")


def normalize_student_key(key: str) -> str:
    """Each prefix is stripped at most once, in the reference's order."""
    for p in _STUDENT_PREFIXES:
        if key.startswith(p):
            key = key[len(p):]
    return key


def merge_student_into_sam3(student_sd: dict, sam3_sd: dict, target_prefix: str = "detector.backbone.vision_backbone.trunk.model.",
                            replace_prefix: str | None = None, skip_teacher_prefixes=()) -> dict:
    """Returns the merged state_dict (`{"model": merged}` is what the reference saves)."""
    prefix = target_prefix.strip(".")
    prefix = f"{prefix}." if prefix else ""
    rep = replace_prefix.strip(".") if replace_prefix is not None else "detector.backbone.vision_backbone.trunk"
    rep = f"{rep}." if rep else ""
    skips = [p.strip(".") + "." for p in skip_teacher_prefixes if p is not None]
    merged = {}
    for k, v in student_sd.items():
        merged[prefix + normalize_student_key(k)] = v
    for k, v in sam3_sd.items():
        if rep and k.startswith(rep):
            continue                                  # the teacher's trunk is replaced by the student
        if any(k.startswith(p) for p in skips) or k in merged:
            continue
        merged[k] = v
    return merged


_TEXT_STUDENT_PREFIXES = ("module.", "detector.backbone.language_backbone.", "backbone.language_backbone.")


def normalize_text_student_key(key: str) -> str:
    for p in _TEXT_STUDENT_PREFIXES:
        if key.startswith(p):
            key = key[len(p):]
    return key


def merge_text_student_into_sam3(student_sd: dict, sam3_sd: dict, target_prefix: str = "detector.backbone.language_backbone.",
                                 replace_prefix: str | None = None, skip_teacher_prefixes=()) -> dict:
    """Returns the merged state_dict; the replace prefix defaults to the target prefix (the SAM3 text encoder's keys)."""
    prefix = target_prefix.strip(".")
    prefix = f"{prefix}." if prefix else ""
    rep = replace_prefix.strip(".") if replace_prefix is not None else target_prefix.strip(".")
    rep = f"{rep}." if rep else ""
    skips = [p.strip(".") + "." for p in skip_teacher_prefixes if p is not None]
    merged = {prefix + normalize_text_student_key(k): v for k, v in student_sd.items()}
    for k, v in sam3_sd.items():
        if (rep and k.startswith(rep)) or any(k.startswith(p) for p in skips) or k in merged:
            continue
        merged[k] = v
    return merged


def clean_merged_keys(sd: dict) -> dict:
    """`_load_checkpoint`'s key clean-up: accepts {'model': sd} or sd."""
    if "model" in sd and isinstance(sd["model"], dict):
        sd = sd["model"]
    out = {}
    for k, v in sd.items():
        if k.startswith("detector."):
            k = k.replace("detector.", "")
        if "student_trunk." in k:
            k = k.replace("student_trunk.", "")
        out[k] = v
    return out
