"""SYNTHIA data directories (reference src/e2eflow/synthia/)."""
