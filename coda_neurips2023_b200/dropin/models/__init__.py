"""`from models import build_model` (reference main.py:20) -> the H100-native model."""
from coda_neurips2023_b200.models import MODEL_FUNCS, build_model  # noqa: F401
from coda_neurips2023_b200.models import helpers, model_3detr, position_embedding, transformer  # noqa: F401
