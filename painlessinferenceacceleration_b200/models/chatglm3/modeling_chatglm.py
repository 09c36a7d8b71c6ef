# -*- coding: utf-8 -*-
"""ChatGLM3 under the reference's import path (models/chatglm3): the same class as models/chatglm."""
from ..chatglm.modeling_chatglm import ChatGLMForConditionalGeneration  # noqa: F401
