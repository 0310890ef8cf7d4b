// dev_block_host.cu -- the pool block owner of gb_internal.cuh (gb_dev_block, gb_dev_carve) on the host, against a pool that
// records what it hands out and takes back.  No device call.  Prints "ok", or the first check that failed.
#include <cstdio>
#include <utility>
#include <vector>

#include "../../glim_b200/csrc/gb_internal.cuh"

static std::vector<std::pair<int, void*>> g_freed;    // (device, block) of every gb_dev_free of a block
static std::vector<std::pair<int, size_t>> g_taken;   // (device, bytes) of every gb_dev_malloc
static char g_mem[4][1024];
void gb_dev_free(int device, void* p) {
  if (p) g_freed.push_back({device, p});
}
cudaError_t gb_dev_malloc(int device, size_t bytes, void** out) {
  *out = g_mem[g_taken.size()];
  g_taken.push_back({device, bytes});
  return cudaSuccess;
}
void gb_set_error(const char*, ...) {}

#define CHECK(c)                                               \
  do {                                                         \
    if (!(c)) {                                                \
      printf("failed: %s (line %d)\n", #c, __LINE__);          \
      return 1;                                                \
    }                                                          \
  } while (0)

int main() {
  int old_block = 0, handle_block = 0;
  // An owner that was never carved (an insert that leaves no voxels) returns the block it takes over from a handle to the
  // pool of its own device, when it ends.
  {
    void* field = &old_block;
    {
      gb_dev_block b(3);
      b.hand_over(field);
      CHECK(field == nullptr && g_freed.empty());
    }
    CHECK(g_freed.size() == 1 && g_freed[0] == std::make_pair(3, (void*)&old_block));
  }
  // The carve measures the layout, takes one block on ctx's device and lays the layout out in it (256-byte aligned takes);
  // after the hand-over the handle holds it and the owner returns the handle's old block.
  g_freed.clear();
  {
    gb_ctx ctx;
    ctx.device = 2;
    gb_dev_block b(2);
    int* a = nullptr;
    double* d = nullptr;
    CHECK(gb_dev_carve(&ctx, b, [&](Carver& cv) {
            a = cv.take<int>(10);
            d = cv.take<double>(3);
          }) == GB_OK);
    CHECK(g_taken.size() == 1 && g_taken[0] == std::make_pair(2, (size_t)512));
    CHECK(b.base == g_mem[0] && (void*)a == g_mem[0] && (char*)d == g_mem[0] + 256);
    void* field = &handle_block;
    b.hand_over(field);
    CHECK(field == g_mem[0] && g_freed.empty());
  }
  CHECK(g_freed.size() == 1 && g_freed[0] == std::make_pair(2, (void*)&handle_block));
  // A move hands the block on; an owner assigned to returns the block it held, to its device.
  g_freed.clear();
  {
    gb_dev_block x(1), y(5);
    x.base = g_mem[1];
    y.base = g_mem[2];
    x = std::move(y);
    CHECK(g_freed.size() == 1 && g_freed[0] == std::make_pair(1, (void*)g_mem[1]));
    CHECK(x.device == 5 && x.base == g_mem[2] && y.base == nullptr);
    gb_dev_block z(std::move(x));
    CHECK(z.device == 5 && z.base == g_mem[2] && x.base == nullptr);
  }
  CHECK(g_freed.size() == 2 && g_freed[1] == std::make_pair(5, (void*)g_mem[2]));
  printf("ok\n");
  return 0;
}
