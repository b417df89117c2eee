/* pwrite_log.c — linked with -Wl,--wrap=pwrite,--wrap=fsync into a test build of the gossip_store file calls: every
 * pwrite's offset and length, and every fsync as offset UINT64_MAX and length 0, in call order, for the test to read
 * back (tests/test_gossip_store_salvage_host.py) */
#define _GNU_SOURCE
#include <stdint.h>
#include <sys/types.h>
#include <unistd.h>

#define LOG_CAP 65536
uint64_t pwrite_log_off[LOG_CAP], pwrite_log_len[LOG_CAP];
size_t pwrite_log_n;

ssize_t __real_pwrite(int fd, const void *buf, size_t count, off_t offset);
ssize_t __wrap_pwrite(int fd, const void *buf, size_t count, off_t offset) {
    if (pwrite_log_n < LOG_CAP) {
        pwrite_log_off[pwrite_log_n] = (uint64_t)offset;
        pwrite_log_len[pwrite_log_n] = count;
    }
    pwrite_log_n++;
    return __real_pwrite(fd, buf, count, offset);
}

int __real_fsync(int fd);
int __wrap_fsync(int fd) {
    if (pwrite_log_n < LOG_CAP) {
        pwrite_log_off[pwrite_log_n] = UINT64_MAX;
        pwrite_log_len[pwrite_log_n] = 0;
    }
    pwrite_log_n++;
    return __real_fsync(fd);
}
