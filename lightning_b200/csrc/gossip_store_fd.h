/* gossip_store_fd.h — the file helpers of gossip_store_fd.c that gossip_salvage_fd.c shares (internal to the library) */
#ifndef GOSSIP_STORE_FD_H
#define GOSSIP_STORE_FD_H
#include <stddef.h>
#include <stdint.h>

#define GSFD_API __attribute__((visibility("hidden")))
/* the checks a file call makes before it reads: SV_OK, or the refusal with errno set (EBADF: not an open descriptor or not
 * open for reading and writing; EINVAL: not a regular file, len 0 or past its end) */
GSFD_API int gsfd_check(int fd, uint64_t len);
/* len bytes from offset 0; -1 with errno on failure (EIO: the file ended early) */
GSFD_API int gsfd_read_all(int fd, uint8_t *p, size_t len);
/* len bytes at offset off; -1 with errno on failure */
GSFD_API int gsfd_write_at(int fd, const uint8_t *p, size_t len, uint64_t off);
/* fsync, retried on EINTR; -1 with errno on failure */
GSFD_API int gsfd_sync(int fd);
#endif
