"""MPI Sintel data directories and inputs (reference src/e2eflow/sintel/)."""
