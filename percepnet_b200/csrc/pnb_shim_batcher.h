// pnb_shim_batcher.h -- group commit of single-frame requests from concurrent threads into one batched call.
//
// Host only, C++11, no dependency on the engine: the call to make is a template parameter, so the batcher compiles on
// its own (tests/test_shim_batcher.py drives it with a mock call).  The pooled rnnoise shim gives every group of
// handles one FrameBatcher whose call is pnb_process_sessions_host_f32 on the group's engine.
//
// process() is synchronous for its caller.  A caller enqueues its request on the FIFO; if no thread is leading, it
// becomes the leader.  The leader repeatedly takes up to `slots` requests in FIFO order, gathers their inputs into one
// [k][frame] buffer (so a request's out may alias its in), drops the lock, makes one call, then scatters out and g/r to
// each request of the batch and marks it done.  Frames that arrive during a call queue up for the next batch.  Once
// its own request is done, the leader hands the lead to the thread of the oldest pending request, or clears it when
// nothing is pending.  There is no helper thread, no timer and no waiting for stragglers: a lone caller makes one call.
//
// Call: int call(const int *ids, int k, const float *in, float *out, float *gr, std::string &err), with in / out
// [k][frame] and gr [k][gr_width]; it returns 0 or an error code and on error fills err.  Every request of a failed
// batch gets the code and the text.  Calls never overlap: only the leader makes them.
#ifndef PNB_SHIM_BATCHER_H
#define PNB_SHIM_BATCHER_H

#include <string.h>

#include <condition_variable>
#include <deque>
#include <mutex>
#include <string>
#include <vector>

namespace pnb {

struct BatcherStats {
  long long calls = 0;    // calls made
  long long frames = 0;   // requests completed (frames advanced, successful or not)
  long long largest = 0;  // largest batch
};

template <class Call>
class FrameBatcher {
 public:
  FrameBatcher(Call call, int slots, int frame, int gr_width)
      : call_(call), slots_(slots), frame_(frame), grw_(gr_width), ids_(slots), in_((size_t)slots * frame),
        out_((size_t)slots * frame), gr_((size_t)slots * gr_width) {}
  FrameBatcher(const FrameBatcher &) = delete;
  FrameBatcher &operator=(const FrameBatcher &) = delete;

  // Returns once this request's out[frame] and gr[gr_width] are written (or its batch failed: then the call's code,
  // with the text in *err when err is not NULL).
  int process(int id, const float *in, float *out, float *gr, std::string *err) {
    Request r;
    r.id = id;
    r.in = in;
    r.out = out;
    r.gr = gr;
    std::unique_lock<std::mutex> lk(mu_);
    q_.push_back(&r);
    if (leading_) {
      while (!r.done && !r.lead) r.cv.wait(lk);
      if (r.done) return finish(r, err);
    }
    leading_ = true;  // taken, or handed over (the flag stays set across a hand-over)
    r.lead = false;
    while (!r.done) run_batch(lk);
    if (!q_.empty()) {
      Request *next = q_.front();
      next->lead = true;
      next->cv.notify_one();
    } else {
      leading_ = false;
    }
    return finish(r, err);
  }

  BatcherStats stats() const {
    std::lock_guard<std::mutex> lk(mu_);
    return stats_;
  }
  // pending requests and whether a leader is marked; both are 0 whenever no process() is running
  int pending() const {
    std::lock_guard<std::mutex> lk(mu_);
    return (int)q_.size();
  }
  bool leading() const {
    std::lock_guard<std::mutex> lk(mu_);
    return leading_;
  }

 private:
  struct Request {
    int id = 0;
    const float *in = nullptr;
    float *out = nullptr;
    float *gr = nullptr;
    bool done = false;
    bool lead = false;
    int rc = 0;
    std::string err;
    std::condition_variable cv;
  };

  static int finish(Request &r, std::string *err) {
    if (r.rc && err) *err = r.err;
    return r.rc;
  }

  // Called with lk held by the leader; returns with lk held.  The queue is never empty here: the leader's own request is
  // pending until a batch completes it.
  void run_batch(std::unique_lock<std::mutex> &lk) {
    const int k = (int)q_.size() < slots_ ? (int)q_.size() : slots_;
    batch_.assign(q_.begin(), q_.begin() + k);
    q_.erase(q_.begin(), q_.begin() + k);
    lk.unlock();
    // the requests' buffers are stable: their callers wait until done is set
    for (int i = 0; i < k; i++) {
      ids_[i] = batch_[i]->id;
      memcpy(&in_[(size_t)i * frame_], batch_[i]->in, (size_t)frame_ * sizeof(float));
    }
    std::string err;
    const int rc = call_(ids_.data(), k, in_.data(), out_.data(), gr_.data(), err);
    if (rc == 0) {
      for (int i = 0; i < k; i++) {
        memcpy(batch_[i]->out, &out_[(size_t)i * frame_], (size_t)frame_ * sizeof(float));
        if (batch_[i]->gr) memcpy(batch_[i]->gr, &gr_[(size_t)i * grw_], (size_t)grw_ * sizeof(float));
      }
    }
    lk.lock();
    stats_.calls++;
    stats_.frames += k;
    if (k > stats_.largest) stats_.largest = k;
    for (int i = 0; i < k; i++) {
      Request *q = batch_[i];
      q->rc = rc;
      if (rc) q->err = err;
      q->done = true;
      q->cv.notify_one();  // under the lock: the waiter cannot return (and destroy q) before it is released
    }
  }

  Call call_;
  const int slots_, frame_, grw_;
  mutable std::mutex mu_;
  std::deque<Request *> q_;
  bool leading_ = false;
  BatcherStats stats_;
  // the leader's working set; only the leader touches it, and leadership passes under mu_
  std::vector<Request *> batch_;
  std::vector<int> ids_;
  std::vector<float> in_, out_, gr_;
};

}  // namespace pnb

#endif  // PNB_SHIM_BATCHER_H
