// How many graph kernel nodes per second does one GPU retire when S host threads replay small graphs on S streams?
// (Question behind it: is the front end with 8 trackers per GPU bound by node dispatch rather than by SM time?)
#include <cuda_runtime.h>
#include <chrono>
#include <cstdio>
#include <thread>
#include <vector>
__global__ void k_spin(long long cycles, int* sink)
{
    const long long t0 = clock64();
    while (clock64() - t0 < cycles) { }
    if (sink && threadIdx.x == 1024) *sink = 1;
}
static void worker(int nodes, int ctas, int threads, long long cycles, int launches, bool fork)
{
    cudaStream_t s, s2; cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking); cudaStreamCreateWithFlags(&s2, cudaStreamNonBlocking);
    cudaEvent_t e1, e2; cudaEventCreateWithFlags(&e1, cudaEventDisableTiming); cudaEventCreateWithFlags(&e2, cudaEventDisableTiming);
    cudaGraph_t g; cudaGraphExec_t ge;
    cudaStreamBeginCapture(s, cudaStreamCaptureModeThreadLocal);
    if (fork) { cudaEventRecord(e1, s); cudaStreamWaitEvent(s2, e1, 0); }
    for (int k = 0; k < nodes; k++) k_spin<<<ctas, threads, 0, (fork && k >= nodes / 2) ? s2 : s>>>(cycles, nullptr);
    if (fork) { cudaEventRecord(e2, s2); cudaStreamWaitEvent(s, e2, 0); }
    cudaStreamEndCapture(s, &g);
    cudaGraphInstantiate(&ge, g, 0);
    for (int i = 0; i < launches; i++) cudaGraphLaunch(ge, s);
    cudaStreamSynchronize(s);
}
// one host thread feeding S streams round-robin (no contention on the driver's locks)
static double single_thread(int S, int nodes, int ctas, int threads, long long cycles, int launches)
{
    std::vector<cudaStream_t> st(S); std::vector<cudaGraphExec_t> ge(S);
    for (int i = 0; i < S; i++) {
        cudaStreamCreateWithFlags(&st[i], cudaStreamNonBlocking);
        cudaGraph_t g;
        cudaStreamBeginCapture(st[i], cudaStreamCaptureModeThreadLocal);
        for (int k = 0; k < nodes; k++) k_spin<<<ctas, threads, 0, st[i]>>>(cycles, nullptr);
        cudaStreamEndCapture(st[i], &g);
        cudaGraphInstantiate(&ge[i], g, 0);
    }
    for (int w = 0; w < 20; w++) for (int i = 0; i < S; i++) cudaGraphLaunch(ge[i], st[i]);
    cudaDeviceSynchronize();
    auto t0 = std::chrono::steady_clock::now();
    for (int w = 0; w < launches; w++) for (int i = 0; i < S; i++) cudaGraphLaunch(ge[i], st[i]);
    const double host = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
    cudaDeviceSynchronize();
    const double sec = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
    printf("   one host thread, S=%2d: %8.0f graphs/s  (host time per launch %.2f us)\n", S, S * launches / sec, 1e6 * host / (S * launches));
    return sec;
}
int main()
{
    cudaFree(0);
    int n_sm = 0;
    cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, 0);
    struct Cfg { int nodes, ctas, threads; long long cycles; bool fork; const char* name; } cfgs[] = {
        {12, 1, 32, 0, false, "12 empty kernels, chain"},
        {12, 1, 32, 0, true, "12 empty kernels, two branches of 6"},
        {12, 1, 256, 10000, false, "12 x (1 CTA, 5 us), chain"},
        {12, 1, 256, 10000, true, "12 x (1 CTA, 5 us), two branches"},
        {12, n_sm, 256, 10000, false, "12 x (one CTA per SM, 5 us), chain"},
        {6, 1, 256, 20000, false, "6 x (1 CTA, 10 us), chain"},
    };
    for (auto& c : cfgs) {
        if (!c.fork) for (int S : {1, 4, 8, 16}) { printf("%-40s", c.name); single_thread(S, c.nodes, c.ctas, c.threads, c.cycles, 1500); }
        for (int S : {1, 2, 4, 8, 16}) {
            const int launches = 1500;
            { std::vector<std::thread> th; for (int i = 0; i < S; i++) th.emplace_back(worker, c.nodes, c.ctas, c.threads, c.cycles, 50, c.fork); for (auto& t : th) t.join(); }
            auto t0 = std::chrono::steady_clock::now();
            std::vector<std::thread> th;
            for (int i = 0; i < S; i++) th.emplace_back(worker, c.nodes, c.ctas, c.threads, c.cycles, launches, c.fork);
            for (auto& t : th) t.join();
            cudaDeviceSynchronize();
            const double sec = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
            printf("%-40s S=%2d: %8.0f graphs/s  %9.0f nodes/s  (%.2f us per graph per stream)\n", c.name, S, S * launches / sec, (double)S * launches * c.nodes / sec, 1e6 * sec / launches);
        }
    }
    return 0;
}
