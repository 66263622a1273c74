// files.cu -- the pinned upload ring (ctx.cuh UploadRing: the context's and each file decoder's) and the status of the corrupt
// files of a file call (k_file_status), which both file decoders (jpeg.cu, png.cu) share
#include "ctx.cuh"

namespace cb200 {

// a picture with corrupt data: status -2 and, on the camera call, no chunks
__global__ void k_file_status(const int* __restrict__ bad, int n, int32_t* __restrict__ status, uint32_t* __restrict__ mask)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n && bad[i]) { status[i] = -2; if (mask) mask[i] = 0; }
}

int file_status(cb200_ctx* c, const int* d_bad, int n, int32_t* d_status, uint32_t* d_mask)
{
    k_file_status<<<(n + 127) / 128, 128, 0, c->stream>>>(d_bad, n, d_status, d_mask);
    count_launch();
    CK(cudaGetLastError(), "status launch");
    return CB200_OK;
}

int UploadRing::take(size_t bytes, int* slot, uint8_t** host)
{
    *slot = next;
    next = (next + 1) % kSlots;
    if (!ev[*slot]) CK(cudaEventCreateWithFlags(&ev[*slot], cudaEventDisableTiming), "cudaEventCreate upload slot");
    CK(cudaEventSynchronize(ev[*slot]), "sync (upload slot)");   // the slot's last copy has run
    CK(h[*slot].ensure(bytes), "cudaMallocHost upload slot");
    *host = h[*slot];
    return CB200_OK;
}

int UploadRing::send(cudaStream_t st, int slot, void* d_dst, size_t bytes)
{
    CK(cudaMemcpyAsync(d_dst, h[slot], bytes, cudaMemcpyHostToDevice, st), "H2D upload");
    CK(cudaEventRecord(ev[slot], st), "record upload slot");
    return CB200_OK;
}

}  // namespace cb200
