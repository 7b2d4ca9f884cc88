// conc_handle.cu -- lifecycle of the ugvc_conc handle (create, free, last error, launch count).  CUB-free, so the
// host emulation (tests/host_emu) can build it together with conc_annotate.cu.
#include "concordance.cuh"

static thread_local std::string g_conc_err;

int conc_fail(ugvc_conc* h, int code, const std::string& msg) {
    if (h) h->err = msg;
    g_conc_err = msg;
    return code;
}

extern "C" int ugvc_conc_create(int device, ugvc_conc** out) {
    ugvc_conc* h = nullptr;
    if (!out) return conc_fail(nullptr, UGVC_E_ARG, "conc_create: out is NULL");
    int n_dev = 0;
    if (cudaGetDeviceCount(&n_dev) != cudaSuccess || n_dev <= 0)
        return conc_fail(nullptr, UGVC_E_CUDA, "conc_create: no CUDA device (there is no CPU path)");
    if (device < 0 || device >= n_dev) return conc_fail(nullptr, UGVC_E_ARG, "conc_create: device out of range");
    h = new ugvc_conc();
    h->device = device;
    if (cudaSetDevice(device) != cudaSuccess || cudaStreamCreate(&h->st) != cudaSuccess) {
        delete h;
        return conc_fail(nullptr, UGVC_E_CUDA, "conc_create: cannot create a stream");
    }
    cudaDeviceGetAttribute(&h->sm_count, cudaDevAttrMultiProcessorCount, device);
    *out = h;
    return UGVC_OK;
}

void conc_drop_curves(ugvc_conc* h) {
    for (int g = 0; g < CONC_GROUPS; ++g) {
        for (int a = 0; a < 3; ++a) {
            if (h->curve[g][a]) cudaFree(h->curve[g][a]);
            h->curve[g][a] = nullptr;
        }
        h->curve_len[g] = 0;
    }
}

void conc_drop_contigs(ugvc_conc* h) {
    for (uint8_t* p : h->annot_seq)
        if (p) cudaFree(p);
    h->annot_seq.clear();
    h->annot_len.clear();
}

extern "C" void ugvc_conc_free(ugvc_conc* h) {
    if (!h) return;
    cudaSetDevice(h->device);
    conc_drop_curves(h);
    conc_drop_contigs(h);
    if (h->st) cudaStreamDestroy(h->st);
    delete h;
}

extern "C" const char* ugvc_conc_last_error(const ugvc_conc* h) { return h ? h->err.c_str() : g_conc_err.c_str(); }
extern "C" long long ugvc_conc_launch_count(const ugvc_conc* h) { return h ? h->launches : 0; }
