"""Cityscapes data directories (reference src/e2eflow/cityscapes/)."""
