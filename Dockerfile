# Operator + runtime image for one 8xH100 box (counterpart of the reference's Dockerfile + build/base/*.Dockerfile:
# there the operator is a distroless Go binary and MPI/sshd live in separate user images; here one image carries the
# daemon, the native launcher, the collective runtime and the example workloads).
#   docker build -t mpi-operator-b200 . && docker run --gpus all --ipc=host --network=host mpi-operator-b200
ARG BASE=nvcr.io/nvidia/pytorch:25.06-py3
FROM ${BASE}
WORKDIR /opt/mpi-operator-b200
COPY . .
RUN make all && python -m compileall -q mpi_operator_b200
ENV PATH=/opt/mpi-operator-b200/mpi_operator_b200/bin:${PATH} \
    PYTHONPATH=/opt/mpi-operator-b200
EXPOSE 8081
ENTRYPOINT ["python", "-m", "mpi_operator_b200.cmd.main"]
# the object API stays on loopback (it can start processes and read Secrets); only /metrics + /healthz are exposed
CMD ["--listen", "127.0.0.1:8087", "--monitoring-port", "8081"]
