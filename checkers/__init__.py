"""Checkers of the native ops that are not restatements of the fp32 reference path (see oracle/ for those)."""
