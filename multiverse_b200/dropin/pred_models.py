# coding=utf-8
"""`import pred_models` for the reference's unchanged callers: re-exports the H100 implementation."""
from multiverse_b200.pred_models import *  # noqa: F401,F403
from multiverse_b200.pred_models import Model, Tester, Trainer, get_model  # noqa: F401
