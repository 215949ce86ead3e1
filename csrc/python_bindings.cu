// python_bindings.cu -- the compiled `flashmoe._C` extension: a thin pybind11 layer over the C-ABI of
// include/flashmoe_b200.h (libflashmoe_b200.so).  Same six functions, argument names and return keys as the reference's
// extension (osayamenja/FlashMoE csrc/python_bindings.cu:194-217):
//
//     moe_forward(input, gate_weights, expert_weights) -> Tensor      reference :17-151
//     initialize() / finalize()                                       reference :157-166
//     get_compiled_config() -> {S, H, E, P, PX, Element_size}         reference :170-179
//     get_bookkeeping() -> {nLx} / get_num_local_experts() -> int     reference :181-189
//
// No torch C++ headers: tensors cross the boundary as Python objects and only their data_ptr / shape / dtype / device are
// read (the C-ABI takes plain pointers), so the extension does not depend on libtorch's ABI.  Differences from the
// reference, all deliberate: errors raise RuntimeError instead of exit(1) (reference debug.cuh:19-43); one call = one
// forward (the reference runs 32 warm-up + 32 timed launches inside moe_forward, :124); the caller's weights are used
// in place (the reference re-uploads every weight on every call, :76-120); rank / world come from the launcher's
// environment (torchrun or OMPI / PMI / SLURM) and the peers' symmetric slabs are mapped through CUDA IPC handles
// exchanged over torch.distributed (replaces nvshmem_init + nvshmem_ptr, reference bootstrap.cuh:295,442-443).
#include <pybind11/pybind11.h>

#include <cstdint>
#include <cstdlib>
#include <stdexcept>
#include <string>
#include <vector>

#include "flashmoe_b200.h"

namespace py = pybind11;

namespace {

fm_ctx_t* g_ctx = nullptr;
fm_dims_t g_dims;
int g_rank = 0, g_world = 1, g_device = 0;

[[noreturn]] void raise_last(const char* what) {
    throw std::runtime_error(std::string(what) + ": " + fm_last_error());
}
void check(int rc, const char* what) {
    if (rc < 0) raise_last(what);
}
void require(bool cond, const std::string& msg) {   // the reference's TORCH_CHECK -> RuntimeError
    if (!cond) throw std::runtime_error(msg);
}

int env_first(std::initializer_list<const char*> names, int dflt) {
    for (const char* n : names) {
        const char* v = std::getenv(n);
        if (v != nullptr && *v) return std::atoi(v);
    }
    return dflt;
}

std::vector<int64_t> shape_of(const py::object& t) {
    std::vector<int64_t> s;
    for (auto d : t.attr("shape")) s.push_back(d.cast<int64_t>());
    return s;
}

void check_tensor(const py::object& t, const char* name) {
    py::module_ torch = py::module_::import("torch");
    require(py::isinstance(t, torch.attr("Tensor")), std::string(name) + " must be a torch.Tensor");
    require(t.attr("is_cuda").cast<bool>(), std::string(name) + " must be CUDA tensor");
    require(t.attr("is_contiguous")().cast<bool>(), std::string(name) + " must be contiguous");
    require(t.attr("dtype").equal(torch.attr("bfloat16")),
            std::string(name) + " must be torch.bfloat16 (the compiled Element type)");
    require(t.attr("device").attr("index").cast<int>() == g_device,
            std::string(name) + " is not on this process's GPU " + std::to_string(g_device));
    require(t.attr("data_ptr")().cast<uintptr_t>() % 16 == 0, std::string(name) + " must start on a 16-byte boundary");
}

}  // namespace

// reference python_bindings.cu:157-159 -> flashmoe::initialize (bootstrap.cuh:532-547)
void initialize() {
    require(g_ctx == nullptr, "initialize() called twice");   // the reference asserts the same (bootstrap.cuh:537)
    py::module_ torch = py::module_::import("torch");
    g_rank = env_first({"RANK", "OMPI_COMM_WORLD_RANK", "PMI_RANK", "SLURM_PROCID"}, 0);
    g_world = env_first({"WORLD_SIZE", "OMPI_COMM_WORLD_SIZE", "PMI_SIZE", "SLURM_NTASKS"}, 1);
    const int local = env_first({"LOCAL_RANK", "OMPI_COMM_WORLD_LOCAL_RANK", "SLURM_LOCALID"}, g_rank);
    const int ndev = torch.attr("cuda").attr("device_count")().cast<int>();
    require(ndev > 0, "no CUDA device visible: the MoE forward path has no CPU fallback");
    g_device = local % ndev;
    torch.attr("cuda").attr("set_device")(g_device);
    check(fm_create(nullptr /* the compiled configuration */, g_rank, g_world, g_device, &g_ctx), "fm_create");
    check(fm_get_dims(g_ctx, &g_dims), "fm_get_dims");
    if (g_world > 1) {
        // out-of-band exchange of the symmetric slabs' CUDA IPC handles (plumbing: torch.distributed, any backend)
        py::module_ dist = py::module_::import("torch.distributed");
        if (!dist.attr("is_initialized")().cast<bool>()) {
            py::object dev = torch.attr("device")("cuda", g_device);
            dist.attr("init_process_group")(py::arg("backend") = "cpu:gloo,cuda:nccl", py::arg("rank") = g_rank,
                                            py::arg("world_size") = g_world, py::arg("device_id") = dev);
        }
        char handle[FM_IPC_HANDLE_BYTES];
        check(fm_symm_export(g_ctx, handle), "fm_symm_export");
        py::list gathered;
        for (int i = 0; i < g_world; ++i) gathered.append(py::none());
        dist.attr("all_gather_object")(gathered, py::bytes(handle, FM_IPC_HANDLE_BYTES));
        std::string all;
        for (auto h : gathered) all += h.cast<std::string>();
        require(all.size() == (size_t)g_world * FM_IPC_HANDLE_BYTES, "peers exported handles of different sizes");
        check(fm_symm_attach_ipc(g_ctx, all.data()), "fm_symm_attach_ipc");
        torch.attr("cuda").attr("synchronize")();
        dist.attr("barrier")();   // every rank's slab is mapped before anyone dispatches into it
    }
}

// reference python_bindings.cu:164-166 -> flashmoe::finalize (bootstrap.cuh:561-588)
void finalize() {
    if (g_ctx != nullptr) {
        fm_destroy(g_ctx);
        g_ctx = nullptr;
    }
}

// reference python_bindings.cu:17-151; the checks mirror its TORCH_CHECKs (:22-65)
py::object moe_forward(py::object input, py::object gate_weights, py::object expert_weights) {
    require(g_ctx != nullptr, "Must call initialize() before moe_forward");
    check_tensor(input, "Input");
    check_tensor(gate_weights, "Gate weights");
    check_tensor(expert_weights, "Expert weights");
    const auto xs = shape_of(input), gs = shape_of(gate_weights), es = shape_of(expert_weights);
    require(xs.size() == 3, "Input must be 3D [batch, seq, H]");
    require(xs[0] * xs[1] == g_dims.S, "Input batch*seq must equal compiled S=" + std::to_string(g_dims.S) + ". Got batch=" +
                                           std::to_string(xs[0]) + ", seq=" + std::to_string(xs[1]));
    require(xs[2] == g_dims.H, "Input hidden_size must equal compiled H=" + std::to_string(g_dims.H));
    require(gs.size() == 2 && gs[0] == g_dims.H && gs[1] == g_dims.E,
            "Gate weights must be [H=" + std::to_string(g_dims.H) + ", E=" + std::to_string(g_dims.E) + "]");
    require(es.size() == 4 && es[0] == g_dims.num_local_experts,
            "Expert count mismatch. Expected " + std::to_string(g_dims.num_local_experts) + " local experts");
    // the context is the compiled configuration's: SwiGLU experts (hidden_act 2) are [nLx, 3, P, H]
    fm_config_t cfg;
    check(fm_compiled_config(&cfg), "fm_compiled_config");
    const int64_t mats = cfg.hidden_act == 2 ? 3 : 2;
    require(es[1] == mats, mats == 2 ? "Expert weights must have up and down projections [nLx, 2, P, H]"
                                     : "SwiGLU expert weights must have gate, up and down projections [nLx, 3, P, H]");
    require(es[2] == g_dims.P && es[3] == g_dims.H,
            "Expert weights must be [*, " + std::to_string(mats) + ", P=" + std::to_string(g_dims.P) +
                ", H=" + std::to_string(g_dims.H) + "]");
    py::module_ torch = py::module_::import("torch");
    py::object out = torch.attr("empty_like")(input);   // freshly allocated, caller-owned (reference :131-148)
    const auto stream = torch.attr("cuda").attr("current_stream")().attr("cuda_stream").cast<uintptr_t>();
    auto ptr = [](const py::object& t) { return reinterpret_cast<void*>(t.attr("data_ptr")().cast<uintptr_t>()); };
    check(fm_moe_forward(g_ctx, ptr(input), ptr(gate_weights), ptr(expert_weights), nullptr, nullptr, ptr(out),
                         reinterpret_cast<void*>(stream)),
          "fm_moe_forward");
    // blocking, like the reference (cudaStreamSynchronize before return, :145); then surface in-kernel protocol timeouts
    torch.attr("cuda").attr("current_stream")().attr("synchronize")();
    check(fm_check(g_ctx), "fm_check");
    return out;
}

// reference python_bindings.cu:170-179
py::dict get_compiled_config() {
    py::dict result;
    if (g_ctx != nullptr) {
        result["S"] = g_dims.S; result["H"] = g_dims.H; result["E"] = g_dims.E; result["P"] = g_dims.P;
        result["PX"] = g_dims.PX; result["Element_size"] = g_dims.element_size;
        return result;
    }
    fm_config_t c;
    check(fm_compiled_config(&c), "fm_compiled_config");
    result["S"] = c.sequence_len * c.mini_batch;
    result["H"] = c.hidden_size;
    result["E"] = c.num_experts;
    result["P"] = c.intermediate_size;
    result["PX"] = (c.num_experts + 63) / 64 * 64;   // reference types.cuh:480
    result["Element_size"] = 2;
    return result;
}

// reference python_bindings.cu:181-185
py::dict get_bookkeeping() {
    require(g_ctx != nullptr, "Must call initialize() first");
    py::dict result;
    result["nLx"] = g_dims.num_local_experts;
    return result;
}

// reference python_bindings.cu:187-189
int get_num_local_experts() {
    require(g_ctx != nullptr, "Must call initialize() first");
    return g_dims.num_local_experts;
}

PYBIND11_MODULE(_C, m) {
    m.doc() = "FlashMoE (H100): fused distributed MoE forward in a single sm_90a kernel";
    m.def("moe_forward", &moe_forward, "MoE forward pass. Tensors must match compiled config dimensions.",
          py::arg("input"), py::arg("gate_weights"), py::arg("expert_weights"));
    m.def("initialize", &initialize, "Create this process's context for the compiled configuration and map the peers");
    m.def("finalize", &finalize, "Release the context");
    m.def("get_compiled_config", &get_compiled_config, "Get compile-time configuration values");
    m.def("get_bookkeeping", &get_bookkeeping, "Get internal bookkeeping values");
    m.def("get_num_local_experts", &get_num_local_experts, "Get the number of local experts");
    m.def("is_initialized", []() { return g_ctx != nullptr; });
    m.def("version", []() { return std::string(fm_version()); });
}
