"""Native CPU components: mpirun (csrc/spawner/mpirun.cc), libmpi shim + pi, shm rendezvous,
launch env contract, OpenAPI/CRD generation, entrypoint.sh."""
import json
import os
import subprocess
import sys

import pytest

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BIN = os.path.join(REPO, "mpi_operator_b200", "bin")
MPIRUN = os.path.join(BIN, "mpirun")
pytestmark = pytest.mark.skipif(not os.path.exists(MPIRUN), reason="native binaries not built (run make)")


def run(args, env=None, timeout=60):
    e = dict(os.environ)
    e.pop("OMPI_MCA_orte_default_hostfile", None)
    e.update(env or {})
    return subprocess.run(args, env=e, capture_output=True, text=True, timeout=timeout)


def test_mpirun_rank_env_all_dialects_and_flags():
    r = run([MPIRUN, "--allow-run-as-root", "-np", "3", "-bind-to", "none", "-map-by", "slot", "-x", "FOO=bar", "-x", "PATH",
             "-mca", "pml", "ob1", "-mca", "btl", "^openib", "--tag-output", "sh", "-c",
             "echo $OMPI_COMM_WORLD_RANK/$OMPI_COMM_WORLD_SIZE $PMI_RANK/$PMI_SIZE $RANK/$WORLD_SIZE $HOROVOD_RANK $LOCAL_RANK "
             "$FOO $OMPI_MCA_pml $OMPI_MCA_btl $K_MPI_JOB_ROLE $MASTER_ADDR"])
    assert r.returncode == 0, r.stderr
    lines = sorted(r.stdout.strip().splitlines())
    assert lines == [f"[1,{i}]<stdout>:{i}/3 {i}/3 {i}/3 {i} {i} bar ob1 ^openib worker 127.0.0.1" for i in range(3)]


def test_mpirun_mpmd_output_files_and_timestamps(tmp_path):
    """MPMD application contexts (`prog1 : -np 2 prog2`, Open MPI / Hydra), per-context -np / -x, MPI_APPNUM in the environment,
    -output-filename DIR (DIR/1/rank.<N>/{stdout,stderr}) and -timestamp-output."""
    out = tmp_path / "logs"
    r = run([MPIRUN, "-np", "1", "--tag-output", "-output-filename", str(out), "sh", "-c",
             "echo master $OMPI_COMM_WORLD_RANK/$OMPI_COMM_WORLD_SIZE app=$PMI_APPNUM role=[$ROLE]", ":",
             "-np", "2", "-x", "ROLE=w", "sh", "-c", "echo worker $PMI_RANK/$PMI_SIZE app=$OMPI_MCA_orte_app_num role=[$ROLE]; echo oops >&2"])
    assert r.returncode == 0, r.stderr
    assert sorted(r.stdout.strip().splitlines()) == ["[1,0]<stdout>:master 0/3 app=0 role=[]", "[1,1]<stdout>:worker 1/3 app=1 role=[w]",
                                                     "[1,2]<stdout>:worker 2/3 app=1 role=[w]"]
    assert (out / "1" / "rank.0" / "stdout").read_text() == "master 0/3 app=0 role=[]\n"
    assert (out / "1" / "rank.2" / "stdout").read_text() == "worker 2/3 app=1 role=[w]\n"
    assert (out / "1" / "rank.1" / "stderr").read_text() == "oops\n"
    src = tmp_path / "appnum.c"
    src.write_text('#include <mpi.h>\n#include <stdio.h>\nint main(int c, char** v) { MPI_Init(&c, &v); int r, f = 0, *a = 0, *u = 0; '
                   'MPI_Comm_rank(MPI_COMM_WORLD, &r); MPI_Comm_get_attr(MPI_COMM_WORLD, MPI_APPNUM, &a, &f); '
                   'MPI_Comm_get_attr(MPI_COMM_WORLD, MPI_UNIVERSE_SIZE, &u, &f); printf("rank %d appnum %d universe %d\\n", r, *a, *u); '
                   'MPI_Finalize(); return 0; }\n')
    exe = tmp_path / "appnum"
    subprocess.run(["gcc", "-I" + os.path.join(REPO, "mpi_operator_b200/include"), "-o", str(exe), str(src), "-L" + os.path.join(REPO, "mpi_operator_b200/lib"),
                    "-lmpi", "-Wl,-rpath," + os.path.join(REPO, "mpi_operator_b200/lib")], check=True)
    r = run([MPIRUN, "-np", "1", str(exe), ":", "-np", "2", str(exe)])
    assert sorted(r.stdout.strip().splitlines()) == ["rank 0 appnum 0 universe 3", "rank 1 appnum 1 universe 3", "rank 2 appnum 1 universe 3"], r.stdout + r.stderr
    r = run([MPIRUN, "-np", "1", "--timestamp-output", "echo", "stamped"])
    import re
    assert re.fullmatch(r"\w{3} \w{3} \d{2} \d{2}:\d{2}:\d{2} \d{4}<stdout>:stamped\n", r.stdout), r.stdout
    r = run([MPIRUN, "-np", "1", "true", ":"])
    assert r.returncode != 0 and "no program after ':'" in r.stderr


def test_mpirun_stdin_routing_merged_stderr_and_output_directory(tmp_path):
    """Open MPI's stdio rules: only rank 0 (or `-stdin RANK`) reads the launcher's stdin, the other ranks see /dev/null;
    `-merge-stderr-to-stdout`; `-output-directory` (the newer spelling of -output-filename); `-pernode`; options that only make
    sense with daemons are accepted silently."""
    reader = "read x; echo r$OMPI_COMM_WORLD_RANK=[$x]"
    r = subprocess.run([MPIRUN, "-np", "2", "sh", "-c", reader], input="hello\n", capture_output=True, text=True, timeout=60)
    assert sorted(r.stdout.split()) == ["r0=[hello]", "r1=[]"], r.stdout + r.stderr
    r = subprocess.run([MPIRUN, "-np", "2", "--stdin", "1", "sh", "-c", reader], input="hello\n", capture_output=True, text=True, timeout=60)
    assert sorted(r.stdout.split()) == ["r0=[]", "r1=[hello]"], r.stdout + r.stderr
    r = subprocess.run([MPIRUN, "-np", "2", "--stdin", "none", "sh", "-c", reader], input="hello\n", capture_output=True, text=True, timeout=60)
    assert sorted(r.stdout.split()) == ["r0=[]", "r1=[]"]
    out = tmp_path / "o"
    r = run([MPIRUN, "-np", "2", "--merge-stderr-to-stdout", "--tag-output", "--output-directory", str(out), "--use-hwthread-cpus", "--verbose",
             "--report-uri", "-", "sh", "-c", "echo to-err >&2"])
    assert r.returncode == 0 and r.stderr == "" and sorted(r.stdout.splitlines()) == ["[1,0]<stdout>:to-err", "[1,1]<stdout>:to-err"], r.stdout + r.stderr
    assert (out / "1" / "rank.1" / "stdout").read_text() == "to-err\n"
    r = run([MPIRUN, "--pernode", "-H", "a,b,c", "sh", "-c", "echo $OMPI_COMM_WORLD_SIZE"])
    assert r.stdout.split() == ["3", "3", "3"], r.stdout + r.stderr


def test_mpirun_hostfile_dialects_and_slot_placement(tmp_path):
    hf = tmp_path / "hostfile"
    hf.write_text("job-worker-0.job.ns.svc slots=2\njob-worker-1.job.ns.svc slots=2\n")
    r = run([MPIRUN, "--hostfile", str(hf), "sh", "-c", "echo $OMPI_COMM_WORLD_RANK $B200MPI_HOSTNAME $OMPI_COMM_WORLD_LOCAL_RANK $OMPI_COMM_WORLD_LOCAL_SIZE"])
    assert sorted(r.stdout.split("\n")[:-1]) == ["0 job-worker-0 0 2", "1 job-worker-0 1 2", "2 job-worker-1 0 2", "3 job-worker-1 1 2"]
    hydra = tmp_path / "hydra"
    hydra.write_text("a.b.c:1\nd.e.f:1\n")
    r = run([MPIRUN, "sh", "-c", "echo $PMI_RANK $B200MPI_HOSTNAME"], env={"HYDRA_HOST_FILE": str(hydra)})
    assert sorted(r.stdout.split()) == sorted("0 a 1 d".split())
    r = run([MPIRUN, "sh", "-c", "echo $PMI_SIZE"], env={"I_MPI_HYDRA_HOST_FILE": str(hydra), "I_MPI_PERHOST": "3"})
    assert r.stdout.split() == ["2", "2"]  # explicit host:n wins over I_MPI_PERHOST


def test_mpirun_gpu_pinning_from_slots_file(tmp_path):
    hf = tmp_path / "hostfile"
    hf.write_text("j-worker-0.j.d.svc slots=1\nj-worker-1.j.d.svc slots=1\n")
    slots = tmp_path / "slots.json"
    slots.write_text(json.dumps({"hosts": {"j-worker-0": [3], "j-worker-1": [5]}}))
    r = run([MPIRUN, "--hostfile", str(hf), "sh", "-c", "echo $RANK $LOCAL_RANK $CUDA_VISIBLE_DEVICES $B200MPI_GPU"],
            env={"B200MPI_SLOTS_FILE": str(slots), "CUDA_VISIBLE_DEVICES": "", "NVIDIA_VISIBLE_DEVICES": ""})
    assert sorted(r.stdout.strip().splitlines()) == ["0 0 3,5 3", "1 1 3,5 5"]


def _fake_sysfs(root, cpus_per_node, gpu_nodes):
    """Two-socket style topology under `root` (B200MPI_SYSFS_ROOT): NUMA nodes with CPU lists, GPUs with their bus ids / numa_node."""
    for n, cpus in enumerate(cpus_per_node):
        d = root / "sys/devices/system/node" / f"node{n}"
        d.mkdir(parents=True)
        (d / "cpulist").write_text(cpus + "\n")
    for k, node in enumerate(gpu_nodes):
        bus = f"0000:{0x1b + 0x20 * k:02X}:00.0"
        (root / "proc/driver/nvidia/gpus" / bus).mkdir(parents=True)
        d = root / "sys/bus/pci/devices" / bus.lower()
        d.mkdir(parents=True)
        (d / "numa_node").write_text(f"{node}\n")


@pytest.mark.skipif(len(os.sched_getaffinity(0)) < 4, reason="needs 4 schedulable CPUs")
def test_mpirun_processor_binding_follows_the_gpus_numa_node(tmp_path):
    """--bind-to none|numa|core, PE=, --cpu-set, --report-bindings (Open MPI's options; the reference's command lines pass
    `-bind-to none`, tensorflow-benchmarks.yaml:23-24, which stays the default): numa = the CPUs next to the rank's GPU."""
    cpus = sorted(os.sched_getaffinity(0))[:4]
    lo, hi = f"{cpus[0]},{cpus[1]}", f"{cpus[2]},{cpus[3]}"
    _fake_sysfs(tmp_path, [lo, hi], [0, 0, 1, 1])
    show = "echo $RANK $(grep Cpus_allowed_list /proc/self/status | cut -f2) $B200MPI_BOUND_NUMA"
    allc = open("/proc/self/status").read().split("Cpus_allowed_list:")[1].split()[0]
    env = {"B200MPI_SYSFS_ROOT": str(tmp_path), "CUDA_VISIBLE_DEVICES": ""}

    def ranks(*flags, np="4", extra=None):
        r = run([MPIRUN, "-np", np, "--oversubscribe", *flags, "sh", "-c", show], env={**env, **(extra or {})})
        return [ln.split()[1:] for ln in sorted(r.stdout.strip().splitlines())], r.stderr

    def fmt(*c):   # the kernel's list format for the chosen CPUs
        c = sorted(c)
        return f"{c[0]}-{c[-1]}" if len(c) > 1 and c[-1] - c[0] == len(c) - 1 else ",".join(map(str, c))
    got, err = ranks("-bind-to", "none", "--report-bindings")
    assert got == [[allc]] * 4 and err.count("is not bound") == 4
    got, err = ranks("--bind-to", "numa", "--report-bindings")
    assert got == [[fmt(*cpus[:2]), "0"]] * 2 + [[fmt(*cpus[2:]), "1"]] * 2
    assert err.count("bound to NUMA node 0") == 2 and err.count("bound to NUMA node 1") == 2
    got, _ = ranks("--bind-to", "core")
    assert [g[0] for g in got] == [str(c) for c in cpus]                        # one core each, next to the own GPU
    got, _ = ranks("--map-by", "numa:PE=2", np="2", extra={"CUDA_VISIBLE_DEVICES": "2,0"})   # PE= implies core binding; GPU order from the environment
    assert got == [[fmt(*cpus[2:]), "1"], [fmt(*cpus[:2]), "0"]]
    got, _ = ranks("--map-by", "numa:PE=2", "--bind-to", "none", np="2")          # an explicit policy wins over PE=
    assert got == [[allc]] * 2
    got, _ = ranks("--bind-to", "socket", "--cpu-set", f"{cpus[1]},{cpus[3]}")
    assert got == [[str(cpus[1]), "0"]] * 2 + [[str(cpus[3]), "1"]] * 2
    got, _ = ranks(np="2", extra={"B200MPI_BIND_TO": "numa"})                     # operator-wide default through the environment
    assert got == [[fmt(*cpus[:2]), "0"]] * 2
    # no GPU information at all: ranks are spread over the NUMA nodes in blocks
    bare = tmp_path / "bare"
    _fake_sysfs(bare, [lo, hi], [])
    r = run([MPIRUN, "-np", "4", "--oversubscribe", "--bind-to", "numa", "sh", "-c", show], env={**env, "B200MPI_SYSFS_ROOT": str(bare)})
    assert [ln.split()[2] for ln in sorted(r.stdout.strip().splitlines())] == ["0", "0", "1", "1"]
    r = subprocess.run([MPIRUN, "-np", "1", "--bind-to", "sideways", "true"], capture_output=True, text=True)
    assert r.returncode != 0 and "unknown -bind-to policy" in r.stderr


def test_mpirun_failure_propagation_kills_siblings_and_reports():
    r = run([MPIRUN, "-np", "3", "sh", "-c", "if [ $RANK = 1 ]; then echo dying >&2; exit 7; fi; sleep 30"], timeout=20)
    assert r.returncode == 7 and "dying" in r.stderr and "exited with non-zero status" in r.stderr
    r = run([MPIRUN, "-np", "1", "/definitely/not/here"])
    assert r.returncode == 127


def test_mpirun_removes_the_jobs_shared_memory_segments(tmp_path):
    """Ranks that crash, get killed or simply exit without MPI_Finalize leave their rendezvous segments behind; the launcher
    removes everything that carries its job id once all ranks are gone."""
    src = tmp_path / "leaky.c"
    src.write_text('#include <mpi.h>\n#include <unistd.h>\nint main(int c, char** v) { MPI_Init(&c, &v); MPI_Barrier(MPI_COMM_WORLD); _exit(0); }\n')
    exe = tmp_path / "leaky"
    subprocess.run(["gcc", "-I" + os.path.join(REPO, "mpi_operator_b200/include"), "-o", str(exe), str(src), "-L" + os.path.join(REPO, "mpi_operator_b200/lib"),
                    "-lmpi", "-Wl,-rpath," + os.path.join(REPO, "mpi_operator_b200/lib")], check=True)
    r = run([MPIRUN, "-np", "3", str(exe)], env={"B200MPI_JOB_ID": "leak-check-job"})
    assert r.returncode == 0, r.stderr
    assert not [n for n in os.listdir("/dev/shm") if "leak-check-job" in n]


def test_mpirun_image_relative_path_falls_back_to_path_lookup():
    r = run([MPIRUN, "-n", "2", "/home/mpiuser/pi", "20000"], env={"PATH": BIN + os.pathsep + os.environ["PATH"], "B200MPI_JOB_ID": f"t-{os.getpid()}"})
    assert r.returncode == 0 and "pi is approximately 3." in r.stdout


def test_libmpi_collectives_via_c_program(tmp_path):
    src = tmp_path / "t.c"
    src.write_text(r'''
#include <mpi.h>
#include <stdio.h>
#include <string.h>
int main(int argc, char** argv) {
  MPI_Init(&argc, &argv);
  int r, n; MPI_Comm_rank(MPI_COMM_WORLD, &r); MPI_Comm_size(MPI_COMM_WORLD, &n);
  double x = r + 1.0, s = 0; MPI_Allreduce(&x, &s, 1, MPI_DOUBLE, MPI_SUM, MPI_COMM_WORLD);
  int mx = r, gmx = -1; MPI_Reduce(&mx, &gmx, 1, MPI_INT, MPI_MAX, 0, MPI_COMM_WORLD);
  char big[200000]; memset(big, r == 2 ? 'z' : 'a', sizeof big); MPI_Bcast(big, sizeof big, MPI_CHAR, 2, MPI_COMM_WORLD);
  int all[16]; MPI_Allgather(&r, 1, MPI_INT, all, 1, MPI_INT, MPI_COMM_WORLD);
  long long v = 5; MPI_Allreduce(MPI_IN_PLACE, &v, 1, MPI_LONG_LONG, MPI_PROD, MPI_COMM_WORLD);
  MPI_Barrier(MPI_COMM_WORLD);
  int ok = (s == n * (n + 1) / 2.0) && big[199999] == 'z' && all[n - 1] == n - 1 && (r != 0 || gmx == n - 1) && v == 625;
  printf("rank %d ok=%d\n", r, ok);
  MPI_Finalize();
  return ok ? 0 : 1;
}''')
    exe = tmp_path / "t"
    inc, lib = os.path.join(REPO, "mpi_operator_b200", "include"), os.path.join(REPO, "mpi_operator_b200", "lib")
    subprocess.run(["gcc", "-O1", f"-I{inc}", str(src), "-o", str(exe), f"-L{lib}", "-lmpi", f"-Wl,-rpath,{lib}"], check=True)
    r = run([MPIRUN, "-np", "4", str(exe)], env={"B200MPI_JOB_ID": f"libmpi-{os.getpid()}"})
    assert r.returncode == 0, r.stdout + r.stderr
    assert sorted(r.stdout.strip().splitlines()) == [f"rank {i} ok=1" for i in range(4)]


def test_launch_env_contract_roundtrip():
    from mpi_operator_b200.launch.env import build_rank_env, rank_info_from_env
    e = build_rank_env(rank=3, world_size=8, local_rank=1, local_size=2, node_rank=1, job_id="ns.job", gpu=5)
    for k in ("OMPI_COMM_WORLD_RANK", "PMI_RANK", "RANK", "HOROVOD_RANK", "B200MPI_RANK"):
        assert e[k] == "3"
    assert e["K_MPI_JOB_ROLE"] == "worker" and e["B200MPI_GPU"] == "5"
    info = rank_info_from_env(e)
    assert (info.rank, info.world_size, info.local_rank, info.local_size, info.job_id) == (3, 8, 1, 2, "ns.job")
    assert rank_info_from_env({"PMI_RANK": "2", "PMI_SIZE": "4", "MPI_LOCALRANKID": "0"}).rank == 2  # Hydra dialect alone
    assert rank_info_from_env({"MASTER_PORT": "29500", "RANK": "1", "WORLD_SIZE": "2"}).job_id.startswith("torch-127.0.0.1-29500")


def test_openapi_crd_and_generated_files_are_current():
    from mpi_operator_b200.api import openapi
    crd = openapi.crd()
    v = crd["spec"]["versions"][0]
    assert crd["spec"]["scope"] == "Namespaced" and v["served"] and v["storage"] and v["subresources"] == {"status": {}}
    spec = v["schema"]["openAPIV3Schema"]["properties"]["spec"]
    assert spec["required"] == ["mpiReplicaSpecs"]
    assert spec["properties"]["mpiImplementation"]["enum"] == ["OpenMPI", "Intel", "MPICH"] and spec["properties"]["mpiImplementation"]["default"] == "OpenMPI"
    assert spec["properties"]["slotsPerWorker"]["default"] == 1 and spec["properties"]["sshAuthMountPath"]["default"] == "/root/.ssh"
    assert spec["properties"]["runPolicy"]["properties"]["suspend"]["default"] is False
    conds = v["schema"]["openAPIV3Schema"]["properties"]["status"]["properties"]["conditions"]
    assert conds["x-kubernetes-list-type"] == "map" and conds["x-kubernetes-list-map-keys"] == ["type"]
    assert len(openapi.swagger()["definitions"]) == 9
    assert subprocess.run([sys.executable, os.path.join(REPO, "hack/generate.py"), "--verify"]).returncode == 0
    assert subprocess.run([sys.executable, os.path.join(REPO, "hack/gen_sdk.py")], capture_output=True).returncode == 0


def test_entrypoint_waits_for_slot_map(tmp_path):
    hf = tmp_path / "hostfile"
    hf.write_text("j-worker-0.j.d.svc:1\n")
    slots = tmp_path / "slots.json"
    slots.write_text('{"hosts": {"j-worker-0": [0]}}')
    ep = os.path.join(REPO, "build/base/entrypoint.sh")
    r = run(["bash", ep, "echo", "started"], env={"K_MPI_JOB_ROLE": "launcher", "HYDRA_HOST_FILE": str(hf), "B200MPI_SLOTS_FILE": str(slots)})
    assert r.returncode == 0 and r.stdout.strip() == "started"
    slots.write_text('{"hosts": {"other": [0]}}')
    r = run(["bash", ep, "echo", "started"], env={"K_MPI_JOB_ROLE": "launcher", "HYDRA_HOST_FILE": str(hf), "B200MPI_SLOTS_FILE": str(slots),
                                                  "B200MPI_ENTRYPOINT_RETRIES": "3"}, timeout=60)
    assert r.returncode != 0 and "never became ready" in r.stderr


@pytest.mark.skipif(not os.path.exists("/usr/bin/g++"), reason="system g++ with libasan not present")
def test_host_runtime_is_clean_under_address_and_ub_sanitizers():
    """`make asan` (SURVEY.md §5.2): launcher + shm rendezvous + libmpi shim built with -fsanitize=address,undefined run
    200 rounds of randomly sized collectives on 4 ranks and the pi example; any report makes the rank exit non-zero,
    which mpirun propagates."""
    r = subprocess.run(["make", "asan"], cwd=REPO, capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    assert "mpi_stress: all 200 iterations verified on 4 ranks" in r.stdout
    assert "ERROR: AddressSanitizer" not in r.stderr and "runtime error:" not in r.stderr


def test_wgmma_gemm_library_builds_loads_and_validates_shapes():
    """libb200mpi_gemm.so (csrc/kernels/gemm_bnstats.cu) is cross-compiled for sm_90a by `make`; its shape contract is
    checked on the host: N and K multiples of 64, at most 132 column blocks (one per H100 SM), M below 2^31."""
    from mpi_operator_b200.ops import gemm_bnstats as g
    if not g.LIB_PATH.exists():
        pytest.skip("native libraries not built (run make)")
    assert g.supported(200704, 256, 64) and g.supported(128, 64, 64) and g.supported(50176, 2048, 512)
    assert not g.supported(128, 96, 64) and not g.supported(128, 64, 32) and not g.supported(0, 64, 64) and not g.supported(127, 64, 64)
    assert g.supported(128, 132 * 128, 64) and not g.supported(128, 132 * 128 + 128, 64)
    assert g.lib().b200mpi_gemm_bnstats_partial_floats(256) == 132 * 2 * 256
    sass = subprocess.run(["/usr/local/cuda/bin/cuobjdump", "-sass", str(g.LIB_PATH)], capture_output=True, text=True)
    if sass.returncode == 0:  # the warpgroup tensor-core and TMA instructions are really there
        for mnemonic in ("HGMMA.64x128x16.F32.BF16", "HGMMA.64x64x16.F32.BF16", "UTMALDG", "UTMASTG", "WARPGROUP.ARRIVE"):
            assert mnemonic in sass.stdout, mnemonic


def test_runtime_launch_planning_on_the_host():
    """`make test_comm_host`: algorithm selection thresholds, grid sizing, per-(op, algo) counters -> JSON and argument
    validation of libb200mpi — the parts of csrc/runtime/comm.cc that decide what gets launched, without a GPU."""
    if not os.path.exists(os.path.join(REPO, "mpi_operator_b200/lib/libb200mpi.so")):
        pytest.skip("native libraries not built (run make)")
    r = subprocess.run(["make", "test_comm_host"], cwd=REPO, capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "comm_host_test: all checks passed" in r.stdout, r.stdout[-2000:] + r.stderr[-2000:]


def test_wgmma_descriptors_match_cute():
    """`make test_gmma_desc`: the K-major / 128-byte-swizzle wgmma shared-memory descriptor packed by hand in
    csrc/kernels/gemm_bnstats.cu is bit-identical to what CuTe builds for the same tile (host-only check)."""
    import importlib.util
    spec = importlib.util.find_spec("flashinfer")   # located, not imported
    inc = os.path.join(os.path.dirname(spec.origin), "data", "cutlass", "include") if spec and spec.origin else ""
    if not os.path.exists(os.path.join(inc, "cute", "arch", "mma_sm90_desc.hpp")):
        pytest.skip("CUTLASS/CuTe headers not available")
    r = subprocess.run(["make", "test_gmma_desc"], cwd=REPO, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "gmma_desc_test: descriptors match CuTe" in r.stdout, r.stdout[-2000:] + r.stderr[-2000:]
    assert "MISMATCH" not in r.stdout


def test_point_to_point_protocol_with_host_threads():
    """`make test_p2p_protocol`: the p2p_run_op<> template of csrc/kernels/p2p.cu — the code the kernel runs — instantiated
    with host threads and atomics: ring shifts over ragged sizes, eager sends, back-pressure on the third chunk, several
    messages per peer in one batch, counters carried across batches."""
    if not os.path.exists(os.path.join(REPO, "mpi_operator_b200/lib/libb200mpi.so")):
        pytest.skip("native libraries not built (run make)")
    r = subprocess.run(["make", "test_p2p_protocol"], cwd=REPO, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "p2p_protocol_test: all checks passed" in r.stdout, r.stdout[-2000:] + r.stderr[-2000:]


def test_wgmma_gemm_pipeline_host_model():
    """`make test_gemm_model`: the roles of csrc/kernels/gemm_bnstats.cu (TMA producer warp, two consumer warpgroups) as
    host threads over emulated mbarriers / TMA / wgmma, sharing the kernel's index and phase arithmetic
    (gemm_bnstats_logic.h). Ring wrap-around across tiles, stage release one k-block behind, ragged M, both tile widths, the
    swizzled staging layout, column sums merged over the two warpgroups and partial rows are checked against a plain GEMM."""
    r = subprocess.run(["make", "test_gemm_model"], cwd=REPO, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "gemm_pipeline_model: all cases match" in r.stdout, r.stdout[-2000:] + r.stderr[-2000:]
    assert "MISMATCH" not in r.stdout


def _torch_nccl_path():
    import importlib.util
    spec = importlib.util.find_spec("nvidia.nccl")
    if spec is None or not spec.submodule_search_locations:
        return None
    p = os.path.join(list(spec.submodule_search_locations)[0], "lib", "libnccl.so.2")
    return p if os.path.exists(p) else None


def test_nccl_shim_covers_the_symbols_libnccl_calls_through_its_own_plt():
    """libnccl calls some of its public entry points through the PLT; with the shim preloaded those internal calls land in
    the shim carrying real ncclComm pointers. Every such symbol the shim exports must therefore take the 'foreign handle'
    path (csrc/nccl_shim/nccl_shim.cu: S(), g_in_real). This checks the list has not grown past what the shim knows."""
    real, shim = _torch_nccl_path(), os.path.join(REPO, "mpi_operator_b200/lib/libb200mpi_nccl.so")
    if real is None or not os.path.exists(shim):
        pytest.skip("bundled libnccl or the shim is not available")
    rel = subprocess.run(["objdump", "-R", real], capture_output=True, text=True).stdout
    internal = {ln.split()[-1].split("@")[0] for ln in rel.splitlines() if "JUMP_SLOT" in ln and ln.split()[-1].startswith("nccl")}
    exported = {ln.split()[-1] for ln in subprocess.run(["nm", "-D", "--defined-only", shim], capture_output=True, text=True).stdout.splitlines()
                if ln.split()[-1].startswith("nccl")}
    handled = {"ncclBroadcast", "ncclCommDeregister", "ncclCommGetAsyncError", "ncclCommRegister", "ncclCommWindowDeregister",
               "ncclDevCommDestroy", "ncclGetErrorString", "ncclGetUniqueId", "ncclGetVersion", "ncclMemAlloc", "ncclMemFree"}
    interposed = internal & exported
    assert interposed <= handled, f"libnccl calls {sorted(interposed - handled)} through its PLT: teach the shim to forward them verbatim"


def test_nccl_shim_pass_through_reaches_the_bundled_nccl_on_the_host():
    shim = os.path.join(REPO, "mpi_operator_b200/lib/libb200mpi_nccl.so")
    if _torch_nccl_path() is None or not os.path.exists(shim):
        pytest.skip("bundled libnccl or the shim is not available")
    code = ("import ctypes,os,torch\n"
            "L=ctypes.CDLL(os.environ['SHIM'])\n"
            "buf=ctypes.create_string_buffer(128)\n"
            "assert L.ncclGetUniqueId(buf)==0\n"
            "v=ctypes.c_int(); assert L.ncclGetVersion(ctypes.byref(v))==0\n"
            "print('MARK', buf.raw[32:39]==b'b200mpi', v.value, sum(1 for l in open('/proc/self/maps') if 'libnccl.so' in l)>0)\n")
    outs = {}
    for mode in ("nccl", "auto"):
        env = dict(os.environ, SHIM=shim, LD_PRELOAD=shim, B200MPI_ALGO=mode)
        r = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=300)
        assert r.returncode == 0, r.stderr[-2000:]
        outs[mode] = [ln for ln in r.stdout.splitlines() if ln.startswith("MARK")][0].split()
    assert outs["auto"][1] == "True"                      # own id: minted by the shim, tagged
    assert outs["nccl"][1] == "False" and outs["nccl"][3] == "True"   # forwarded: a real NCCL id, bundled libnccl mapped
    assert int(outs["nccl"][2]) >= 22000


def test_nccl_shim_exports_every_nccl_symbol_torch_imports():
    """LD_PRELOAD only works if no ncclX call of libtorch can slip past the shim into the real library with one of our
    handles: every nccl* symbol libtorch_cuda imports must be defined by libb200mpi_nccl.so."""
    import torch
    shim = os.path.join(REPO, "mpi_operator_b200/lib/libb200mpi_nccl.so")
    lib = os.path.join(os.path.dirname(torch.__file__), "lib", "libtorch_cuda.so")
    if not (os.path.exists(shim) and os.path.exists(lib)):
        pytest.skip("libtorch_cuda.so or the shim is not available")
    need = {ln.split()[-1] for ln in subprocess.run(["nm", "-D", "--undefined-only", lib], capture_output=True, text=True).stdout.splitlines()
            if ln.split() and ln.split()[-1].startswith("nccl")}
    have = {ln.split()[-1] for ln in subprocess.run(["nm", "-D", "--defined-only", shim], capture_output=True, text=True).stdout.splitlines()
            if ln.split() and ln.split()[-1].startswith("nccl")}
    assert need, "libtorch_cuda.so imports no nccl symbols?"
    assert need <= have, f"shim is missing {sorted(need - have)}"


def test_libmpi_point_to_point_and_vector_collectives():
    """`make test_mpi_p2p`: MPI_Send/Recv/Isend/Irecv/Wait/Test/Probe/Sendrecv, Gatherv/Scatterv/Allgatherv, Scan/Exscan,
    Reduce_scatter_block of the libmpi shim on 4 ranks and on 1 rank (csrc/tests/mpi_p2p_test.cc): head-to-head 8 MiB sends
    do not deadlock, an eager send is deliverable before the receiver's first call, same-tag messages do not overtake."""
    r = subprocess.run(["make", "test_mpi_p2p"], cwd=REPO, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    assert "all checks passed on 4 ranks" in r.stdout and "all checks passed on 1 ranks" in r.stdout
