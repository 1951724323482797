// loader_pool.h — the host-side pieces of the file streamer that do not touch CUDA: the streaming copy into the
// page-locked pool and the long-lived loader threads. Header-only so that the CPU test suite can exercise them under
// ThreadSanitizer / AddressSanitizer without a GPU (tests/native/loader_pool_test.cpp).
#pragma once
#include <condition_variable>
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <mutex>
#include <thread>
#include <vector>
#if defined(__x86_64__)
#include <emmintrin.h>
#endif

// Copy with non-temporal stores: the destination lines go to memory without being read or left in the cache.
// The loaders must not fill the page-locked pool with ordinary stores (pread straight into it): each piece would
// stay dirty in the cache of whichever core read it, and the copy engine's reads of such lines are served by
// cross-core snoops — measured on a 2-socket host at ~19 GB/s against ~52 GB/s for lines that
// are in DRAM. Each loader therefore preads into a 256 KB cache-resident staging buffer and streams it out.
static inline void copyStreaming(char* dst, const char* src, uint64_t bytes) {      // dst, src 16-byte aligned, bytes % 16 == 0
#if defined(__x86_64__)
    uint64_t i = 0;
    for (; i + 64 <= bytes; i += 64) {
        __m128i a = _mm_load_si128((const __m128i*)(src + i)), b = _mm_load_si128((const __m128i*)(src + i + 16));
        __m128i c = _mm_load_si128((const __m128i*)(src + i + 32)), d = _mm_load_si128((const __m128i*)(src + i + 48));
        _mm_stream_si128((__m128i*)(dst + i), a); _mm_stream_si128((__m128i*)(dst + i + 16), b);
        _mm_stream_si128((__m128i*)(dst + i + 32), c); _mm_stream_si128((__m128i*)(dst + i + 48), d);
    }
    for (; i < bytes; i += 16) _mm_stream_si128((__m128i*)(dst + i), _mm_load_si128((const __m128i*)(src + i)));
    _mm_sfence();
#else
    memcpy(dst, src, bytes);
#endif
}

// same, source at any alignment (the O_DIRECT path reads whole 4 KB blocks; the records start 24 + 16 k bytes into the file)
static inline void copyStreamingU(char* dst, const char* src, uint64_t bytes) {     // dst 16-byte aligned, bytes % 16 == 0
#if defined(__x86_64__)
    uint64_t i = 0;
    for (; i + 64 <= bytes; i += 64) {
        __m128i a = _mm_loadu_si128((const __m128i*)(src + i)), b = _mm_loadu_si128((const __m128i*)(src + i + 16));
        __m128i c = _mm_loadu_si128((const __m128i*)(src + i + 32)), d = _mm_loadu_si128((const __m128i*)(src + i + 48));
        _mm_stream_si128((__m128i*)(dst + i), a); _mm_stream_si128((__m128i*)(dst + i + 16), b);
        _mm_stream_si128((__m128i*)(dst + i + 32), c); _mm_stream_si128((__m128i*)(dst + i + 48), d);
    }
    for (; i < bytes; i += 16) _mm_stream_si128((__m128i*)(dst + i), _mm_loadu_si128((const __m128i*)(src + i)));
    _mm_sfence();
#else
    memcpy(dst, src, bytes);
#endif
}

// Long-lived loader threads of the file streamer (the reference keeps its loaders alive too, main.cpp:811-958).
// Creating the threads per call was measured at 1.0 ms for 32 and 2.5 ms for 64 threads in a process that holds a
// CUDA context, and retiring them cost more — comparable to the whole read of a 256 MB file.
struct LoaderPool {
    std::vector<std::thread> threads;
    std::mutex m;
    std::condition_variable cvStart, cvDone;
    std::function<void(int)> job;
    std::vector<char*> bounce;        // one cache-resident staging buffer per worker (BOUNCE_BYTES)
    std::vector<char*> direct;        // one 4 KB-aligned block buffer per worker for O_DIRECT reads (DIRECT_BYTES), allocated on first use
    static constexpr size_t BOUNCE_BYTES = 256 << 10;
    static constexpr size_t DIRECT_BYTES = (1 << 20) + 8192;
    char* directBuffer(int idx) {     // called by worker idx only
        if (!direct[idx]) direct[idx] = (char*)aligned_alloc(4096, DIRECT_BYTES);
        return direct[idx];
    }
    uint64_t generation = 0;
    int wanted = 0, running = 0;
    bool quit = false;

    void worker(int idx) {
        uint64_t seen = 0;
        for (;;) {
            std::function<void(int)> fn;
            {
                std::unique_lock<std::mutex> lk(m);
                cvStart.wait(lk, [&] { return quit || generation != seen; });
                if (quit) return;
                seen = generation;
                if (idx >= wanted) continue;
                fn = job;
            }
            fn(idx);
            std::lock_guard<std::mutex> lk(m);
            if (--running == 0) cvDone.notify_all();
        }
    }
    // start n workers on fn; returns at once. fn must stay valid until wait() returns.
    void run(int n, std::function<void(int)> fn) {
        while ((int)threads.size() < n) {
            int idx = (int)threads.size();
            bounce.push_back((char*)aligned_alloc(64, BOUNCE_BYTES));
            direct.push_back(nullptr);
            threads.emplace_back([this, idx] { worker(idx); });
        }
        std::lock_guard<std::mutex> lk(m);
        job = std::move(fn); wanted = n; running = n; generation++;
        cvStart.notify_all();
    }
    void wait() {
        std::unique_lock<std::mutex> lk(m);
        cvDone.wait(lk, [&] { return running == 0; });
    }
    ~LoaderPool() {
        { std::lock_guard<std::mutex> lk(m); quit = true; }
        cvStart.notify_all();
        for (auto& t : threads) t.join();
        for (char* b : bounce) free(b);
        for (char* b : direct) free(b);
    }
};

