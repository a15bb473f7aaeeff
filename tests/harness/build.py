"""Build the glue test harness (tests/harness/_build/*.so).  It is compiled against pgvector's own headers, so it is
built only where a pgvector source tree is present (PGV_REFERENCE, default /root/reference); elsewhere the tests that
need it skip."""
import os
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
REF = os.path.join(os.environ.get("PGV_REFERENCE", "/root/reference"), "src")
EXT = os.path.join(ROOT, "pgvector_b200", "ext")
OUT = os.path.join(HERE, "_build")
SRCS = [os.path.join(HERE, f) for f in ("harness_common.c", "harness_ivf.c", "harness_hnsw.c", "harness_broker.c")] + \
       [os.path.join(EXT, f) for f in ("vb_ivfflat_scan.c", "vb_ivfflat_build.c", "vb_hnsw_scan.c", "vb_hnsw_build.c", "vb_broker.c")] + \
       [os.path.join(EXT, "pgstub", "pgstub_runtime.c")]
FLAGS = ["-std=gnu11", "-O1", "-g", "-fPIC", "-shared", "-pthread", "-Wall", "-Werror", "-Wno-unused-function", "-Wno-comment",
         "-I" + os.path.join(EXT, "pgstub"), "-I" + REF, "-I" + os.path.join(ROOT, "include"), "-I" + EXT, "-I" + HERE]


def paths():
    return os.path.join(OUT, "libvbharness_mock.so"), os.path.join(OUT, "libvbharness_real.so")


def build(force=False):
    mock, real = paths()
    if not os.path.isdir(REF):
        return os.path.exists(mock), os.path.exists(real)
    os.makedirs(OUT, exist_ok=True)
    deps = SRCS + [os.path.join(HERE, f) for f in ("mock_abi.c", "harness_common.h")] + [os.path.join(EXT, "vb_glue.h"), os.path.join(EXT, "vb_broker.h"),
                                                                                        os.path.join(EXT, "pgstub", "postgres.h"),
                                                                                        os.path.join(ROOT, "include", "vecb200.h")]
    newest = max(os.path.getmtime(d) for d in deps)
    import oracle
    oracle.build()
    if force or not os.path.exists(mock) or os.path.getmtime(mock) < newest:
        cmd = ["gcc", *FLAGS, "-o", mock + ".tmp", *SRCS, os.path.join(HERE, "mock_abi.c"),
               "-L" + os.path.join(ROOT, "oracle"), "-l:liboracle.so", "-Wl,-rpath,$ORIGIN/../../../oracle", "-lm"]
        subprocess.run(cmd, check=True, capture_output=True, text=True)
        os.replace(mock + ".tmp", mock)
    lib = os.path.join(ROOT, "pgvector_b200", "libvecb200.so")
    if os.path.exists(lib) and (force or not os.path.exists(real) or os.path.getmtime(real) < newest):
        cmd = ["gcc", *FLAGS, "-o", real + ".tmp", *SRCS, "-L" + os.path.dirname(lib), "-l:libvecb200.so",
               "-Wl,-rpath,$ORIGIN/../../../pgvector_b200", "-lm"]
        subprocess.run(cmd, check=True, capture_output=True, text=True)
        os.replace(real + ".tmp", real)
    return os.path.exists(mock), os.path.exists(real)


if __name__ == "__main__":
    try:
        print(build(force=True))
    except subprocess.CalledProcessError as e:
        print(e.stderr)
        raise
