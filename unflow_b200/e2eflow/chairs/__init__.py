"""FlyingChairs data directories and inputs (reference src/e2eflow/chairs/)."""
