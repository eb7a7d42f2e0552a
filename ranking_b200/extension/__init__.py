"""Premade models of the reference's `tfr.extension.premade`."""
from ranking_b200.extension import tfrbert
