// A library-owned host thread that runs one job at a time for as long as it lives: the compress context's two provers (compress.cu) and
// the compressed verifier's secondary circuit (compress_verify.cu).  The thread keeps its thread-local reduction scratch (sc_scratch.cuh)
// from one job to the next.
#pragma once
#include <condition_variable>
#include <functional>
#include <mutex>
#include <thread>

namespace lurk {

class Worker {
  public:
    Worker() : th_([this] { loop(); }) {}
    ~Worker() {
        { std::lock_guard<std::mutex> g(mu_); stop_ = true; }
        cv_.notify_all();
        th_.join();
    }
    void post(std::function<void()> f) {
        { std::lock_guard<std::mutex> g(mu_); job_ = std::move(f); }
        cv_.notify_all();
    }
    void wait() {
        std::unique_lock<std::mutex> g(mu_);
        cv_.wait(g, [&] { return !job_; });
    }

  private:
    void loop() {
        std::unique_lock<std::mutex> g(mu_);
        for (;;) {
            cv_.wait(g, [&] { return stop_ || job_; });
            if (!job_) return;
            std::function<void()> f = job_;
            g.unlock();
            f();
            g.lock();
            job_ = nullptr;
            cv_.notify_all();
        }
    }
    std::mutex mu_;
    std::condition_variable cv_;
    std::function<void()> job_;
    bool stop_ = false;
    std::thread th_;            // last: the thread starts once the members it uses exist
};

}  // namespace lurk
