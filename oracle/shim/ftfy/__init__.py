"""Tests-only stand-in for ftfy (imported by CLIP/clip/simple_tokenizer.py): the golden prompts are plain ASCII, which fix_text leaves
unchanged."""


def fix_text(text):
    return text
