// engine.cu -- the lifecycle entry points shared by every planned engine (C ABI: include/mi3d.h, "Planned engines"): one handle
// type, one parameter registry (plan::Builder::params) and one weight loader (plan::Builder::load_param and its overrides).
#include "engine_plan.cuh"

namespace {

plan::Builder* builder(mi3d_engine_t h) { return static_cast<plan::Builder*>(h); }   // every engine is a plan::Builder

const plan::Param* param_at(mi3d_engine_t h, int i) {
    if (!h || i < 0 || i >= (int)builder(h)->params.size()) return nullptr;
    return &builder(h)->params[i];
}

}  // namespace

extern "C" {

void mi3d_engine_destroy(mi3d_engine_t h) { delete h; }

int mi3d_engine_num_params(mi3d_engine_t h) { return h ? (int)builder(h)->params.size() : 0; }

const char* mi3d_engine_param_name(mi3d_engine_t h, int i) {
    const plan::Param* P = param_at(h, i);
    return P ? P->name.c_str() : nullptr;
}

int mi3d_engine_param_shape(mi3d_engine_t h, int i, int* shape4) {
    const plan::Param* P = param_at(h, i);
    if (!P || !shape4) return -1;
    for (int k = 0; k < 4; k++) shape4[k] = k < (int)P->shape.size() ? P->shape[k] : 0;
    return (int)P->shape.size();
}

int mi3d_engine_load_param(mi3d_engine_t h, int i, const float* src, const float* partner_src, mi3d_stream_t stream) {
    const plan::Param* P = param_at(h, i);
    if (!P || !src) return MI3D_ERR_ARG;
    return builder(h)->load_param(*P, src, partner_src, (cudaStream_t)stream);
}

int mi3d_engine_set_graph_replay(mi3d_engine_t h, int enable) {
    if (!h) return MI3D_ERR_ARG;
    builder(h)->use_graph = enable != 0;
    return MI3D_OK;
}

int mi3d_engine_graph_replays(mi3d_engine_t h) { return h ? builder(h)->graph_replays() : -1; }

int mi3d_engine_debug_tensor(mi3d_engine_t h, const char* name, void** ptr, size_t* bytes) {
    if (!h || !name || !ptr || !bytes) return MI3D_ERR_ARG;
    const auto& named = builder(h)->named;
    auto it = named.find(name);
    if (it == named.end()) return MI3D_ERR_ARG;
    *ptr = it->second.first; *bytes = it->second.second;
    return MI3D_OK;
}

}  // extern "C"
