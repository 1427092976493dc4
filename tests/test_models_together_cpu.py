"""What tests/test_gpu_models_together.py stands on, checked without a GPU: every kernel's dynamic shared-memory limit is
set through ``set_smem_limit`` (which only ever raises it), and the models of that file land in the TreeSHAP length
buckets it assumes."""

import os
import re

import pytest

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "databricks_kubernetes_mlops_poc_b200", "csrc")
LIMIT = re.compile(r"\bcu(?:da)?FuncSetAttribute\s*\(")


def _code(text: str) -> str:
    """``text`` with its comments blanked (newlines kept, so offsets keep their line numbers)."""
    blank = lambda m: re.sub(r"[^\n]", " ", m.group(0))  # noqa: E731
    return re.sub(r"/\*.*?\*/|//[^\n]*", blank, text, flags=re.S)


def _call_args(code: str, open_paren: int) -> str:
    depth = 0
    for i in range(open_paren, len(code)):
        depth += {"(": 1, ")": -1}.get(code[i], 0)
        if depth == 0:
            return code[open_paren + 1:i]
    raise AssertionError("unbalanced call")


def stray_limit_calls(csrc: str = CSRC):
    """-> (calls inside set_smem_limit, [file:line of every call that sets a dynamic shared-memory limit elsewhere])."""
    inside, stray = 0, []
    for name in sorted(os.listdir(csrc)):
        if not name.endswith((".cu", ".cuh", ".h", ".cpp")):
            continue
        with open(os.path.join(csrc, name)) as f:
            code = _code(f.read())
        body = (-1, -1)
        d = re.search(r"\bset_smem_limit\s*\([^)]*\)\s*\{", code)
        if d:
            depth, i = 0, d.end() - 1
            for i in range(d.end() - 1, len(code)):
                depth += {"{": 1, "}": -1}.get(code[i], 0)
                if depth == 0:
                    break
            body = (d.end(), i)
        for m in LIMIT.finditer(code):
            args = _call_args(code, m.end() - 1)
            if "MaxDynamicSharedMemorySize" not in args and "MAX_DYNAMIC_SHARED_SIZE_BYTES" not in args:
                continue
            if body[0] <= m.start() < body[1]:
                inside += 1
            else:
                stray.append(f"{name}:{code.count(chr(10), 0, m.start()) + 1}")
    return inside, stray


def test_every_shared_memory_limit_goes_through_set_smem_limit():
    """A kernel's dynamic shared-memory limit belongs to the kernel on the device, not to a model: a call that sets it
    straight to one model's need can lower it under another model's launches.  So only set_smem_limit sets it."""
    inside, stray = stray_limit_calls()
    assert inside == 1, "set_smem_limit (csrc/b2f_api.cu) should hold the one cudaFuncSetAttribute of the library"
    assert stray == [], f"dynamic shared-memory limits set outside set_smem_limit: {stray}"


def test_stray_limit_calls_are_found(tmp_path):
    """The guard itself: a direct call (over two lines, after a comment that names the function) is found, and one inside
    a function of another name that merely contains set_smem_limit's name is not taken for the helper."""
    (tmp_path / "a.cuh").write_text(
        "/* cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, 1) in a comment */\n"
        "template <typename K> static cudaError_t set_smem_limit(K kernel, int bytes) {\n"
        "    if (bytes) { return cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes); }\n"
        "    return cudaSuccess;\n"
        "}\n"
        "static int attach(int smem) {\n"
        "    CUDA_TRY(cudaFuncSetAttribute(k_knn_chunk,\n"
        "                                  cudaFuncAttributeMaxDynamicSharedMemorySize, smem));\n"
        "    CUDA_TRY(cudaFuncSetAttribute(k_other, cudaFuncAttributePreferredSharedMemoryCarveout, 50));\n"
        "    return set_smem_limit(k_mmd_row_sums, smem);\n"
        "}\n")
    assert stray_limit_calls(str(tmp_path)) == (1, ["a.cuh:7"])


@pytest.fixture(scope="module")
def tables(curated, rf100d6):
    """The path tables of the GPU file's models A, B, C and D's tiny forest -> their longest path."""
    import schema_zoo as sz

    from databricks_kubernetes_mlops_poc_b200.flatten import flatten_explainer, parse_explainer
    from oracle import reference_pipeline as rp
    from test_gpu_models_together import B_PARAMS, C_PARAMS, SMALL

    pipes = {"A": rf100d6, "B": rp.fit_reference_pipeline(curated.iloc[:6000], B_PARAMS),
             "C": rp.fit_reference_pipeline(curated.iloc[:6000], C_PARAMS)}
    pipes.update({name: sz.fitted(name)[1] for name in SMALL})
    return {name: parse_explainer(flatten_explainer(pipe))["max_len"] for name, pipe in pipes.items()}


def test_models_land_in_the_buckets_the_gpu_tests_assume(tables):
    """B is the suite's one forest in the 16-element bucket; A and the tiny forest share the 9-element bucket (so the tiny
    forest's explainer attach would lower A's limits), and C is in the 24-element bucket."""
    from test_gpu_models_together import bucket

    assert 10 <= tables["B"] <= 16, tables
    assert {n: bucket(v) for n, v in tables.items()} == {"A": 9, "B": 16, "C": 24, "tiny": 9, "packed_wide_gbdt": 9}, tables
